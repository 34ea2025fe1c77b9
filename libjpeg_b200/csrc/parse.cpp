// parse.cpp -- host-side marker parser, restart-interval index and decoder-table builder.
//
// Restates, over a flat in-memory byte view, what the reference does incrementally through its ByteStream:
//   SOI / marker walk          codestream/decoder.cpp:77, codestream/tables.cpp:1003-1420
//   DQT                        marker/quantization.cpp:474-537
//   DHT                        marker/huffmantable.cpp:127-169, coding/huffmantemplate.cpp:878-904
//   DRI                        marker/restartintervalmarker.cpp:80-102
//   SOF0/SOF1                  marker/frame.cpp:111-214, marker/component.cpp:86-111, component.hpp:99-106
//   SOS                        marker/scan.cpp:163-315
//   RSTn sequence              codestream/entropyparser.cpp:117-136, entropyparser.hpp:147-160
//   two-level Huffman decoder  coding/huffmantemplate.cpp:802-874, coding/huffmandecoder.hpp:64-124
// The validation rules and error codes follow those files so that LastError reports what a client of the
// reference would see.
#include <cstdlib>
#include <cstring>

#include "internal.hpp"
#include "specsync.hpp"

namespace b200jpg {

const uint8_t kZigZagToRaster[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                     12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                     35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                     58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

namespace {

struct Cursor {
    const uint8_t *d;
    size_t n;
    int u8(size_t p) const { return p < n ? d[p] : -1; }
    int u16(size_t p) const { return p + 1 < n ? (d[p] << 8) | d[p + 1] : -1; }
};

#define FAIL(code, msg) \
    do {                \
        err = msg;      \
        return code;    \
    } while (0)

// Walks one entropy coded segment, recording every restart marker (position of its 0xff, id byte).
// Returns the offset of the marker that ends the segment -- the first 0xff followed by a byte in c0..ef that is no restart
// marker -- or n. 0xff followed by 01..bf / f0..fe is no marker to EntropyParser::ParseRestartMarker (it eats such bytes while
// it resynchronises, codestream/entropyparser.cpp:191-196); the bit reader of the interval in which they stand stops there
// all the same (io/bitstream.cpp:96-101), which the unstuff kernel reproduces.
size_t index_ecs(const Cursor &c, size_t pos, std::vector<size_t> &rst_at, std::vector<uint8_t> &rst_id) {
    const uint8_t *d = c.d;
    size_t n = c.n;
    while (pos < n) {
        const void *q = memchr(d + pos, 0xff, n - pos);
        if (!q) return n;
        pos = (size_t)((const uint8_t *)q - d);
        if (pos + 1 >= n) return n;
        uint8_t m = d[pos + 1];
        if (m == 0x00) {
            pos += 2;  // stuffed byte
        } else if (m == 0xff) {
            pos += 1;  // fill byte in front of a marker (entropyparser.cpp:121-125)
        } else if (m >= 0xd0 && m <= 0xd7) {
            rst_at.push_back(pos);
            rst_id.push_back(m);
            pos += 2;
        } else if (m >= 0xc0 && m < 0xf0) {
            return pos;
        } else {
            pos += 1;  // garbage
        }
    }
    return n;
}

}  // namespace

// The reference's restart-marker bookkeeping including its resynchronisation (EntropyParser::ParseRestartMarker,
// codestream/entropyparser.cpp:117-199), as a function of the marker sequence alone: the bit reader never passes a marker, so
// when interval k-1 is done the parser stands at, or scans forward to, the first marker behind that interval's data --
//   the expected RSTn                  : consumed, interval k starts behind it;
//   an RSTn that is 4..7 ids "behind"  : dropped together with the data that follows it, the scan goes on;
//   an RSTn that is 1..3 ids "ahead"   : interval k is lost (its MCUs stay cleared), the marker stays for the next interval;
//   any other marker (the segment end) : interval k and everything after it is lost;
//   the end of the data                : UNEXPECTED_EOF.
// off[k] = SIZE_MAX marks a lost interval. Returns 0 or B200JPG_ERR_UNEXPECTED_EOF.
int resolve_restart_sequence(const std::vector<size_t> &rst_at, const std::vector<uint8_t> &rst_id, size_t ecs_off, size_t ecs_end,
                             bool ended_by_eof, std::vector<size_t> &off, std::vector<size_t> &end) {
    const size_t nint = off.size();
    size_t p = 0;  // index of the marker the parser stands at / looks for next
    unsigned next = 0;
    off[0] = ecs_off;
    end[0] = rst_at.empty() ? ecs_end : rst_at[0];
    for (size_t k = 1; k < nint; k++) {
        bool valid = false;
        for (;;) {
            if (p >= rst_at.size()) {  // the marker that ends the segment, or the end of the data
                if (ended_by_eof) return B200JPG_ERR_UNEXPECTED_EOF;
                break;
            }
            const unsigned id = rst_id[p] & 7u;
            if (id == next) {
                off[k] = rst_at[p] + 2;
                p++;
                valid = true;
                break;
            }
            if (((id - next) & 7u) >= 4u) {
                p++;  // behind: drop it and keep looking
                continue;
            }
            break;  // ahead: this interval is lost, the marker stays
        }
        next = (next + 1u) & 7u;
        if (valid) end[k] = p < rst_at.size() ? rst_at[p] : ecs_end;
        else off[k] = SIZE_MAX, end[k] = ecs_end;
    }
    return 0;
}

// Exif (CIPA DC-008): "Exif\0\0", a TIFF header ("II*\0" little endian or "MM\0*" big endian, then the uint32 offset of IFD0
// from the header), IFD0 = a 2-byte entry count and 12-byte entries {tag, type, count, value or offset}. Orientation is tag
// 0x0112, type 3 (SHORT), count 1, its value in the first two bytes of the value field. Only what lies inside the segment is
// read; IFD1, XMP and every other tag are ignored.
int exif_orientation_of(const uint8_t *s, size_t rem) {
    if (rem < 6 || memcmp(s, "Exif\0\0", 6) != 0) return 0;
    const uint8_t *t = s + 6;
    const uint64_t tlen = rem - 6;
    if (tlen < 8) return 1;
    bool le;
    if (memcmp(t, "II*\0", 4) == 0) le = true;
    else if (memcmp(t, "MM\0*", 4) == 0) le = false;
    else return 1;
    auto u16 = [&](uint64_t p) -> uint32_t { return le ? (t[p] | (t[p + 1] << 8)) : ((t[p] << 8) | t[p + 1]); };
    auto u32 = [&](uint64_t p) -> uint32_t { return le ? (u16(p) | (u16(p + 2) << 16)) : ((u16(p) << 16) | u16(p + 2)); };
    const uint64_t ifd = u32(4);
    if (ifd + 2 > tlen) return 1;
    const uint32_t count = u16(ifd);
    for (uint64_t k = 0; k < count; k++) {
        const uint64_t e = ifd + 2 + 12 * k;
        if (e + 12 > tlen) return 1;
        if (u16(e) != 0x0112) continue;
        if (u16(e + 2) != 3 || u32(e + 4) != 1) return 1;
        const uint32_t v = u16(e + 8);
        return (v >= 1 && v <= 8) ? (int)v : 1;
    }
    return 1;
}

int parse_codestream(const uint8_t *data, size_t len, ParsedFrame &out, std::string &err, bool device_index) {
    Cursor c{data, len};
    b200jpg_frame_info &fi = out.info;
    memset(&fi, 0, sizeof(fi));
    out.scans.clear();
    out.orientation = 1;
    out.adobe_transform = -1;
    bool exif_seen = false;  // the first Exif segment decides
    if (!data || len < 4) FAIL(B200JPG_ERR_UNEXPECTED_EOF, "stream is too short to be a JPEG codestream");
    if (c.u16(0) != 0xffd8) FAIL(B200JPG_ERR_MALFORMED_STREAM, "stream does not start with SOI, not a JPEG codestream");

    HuffSpec dc[4], ac[4];
    uint16_t quant[4][64];
    bool quant_defined[4] = {false, false, false, false};
    uint32_t dri = 0;
    bool have_sof = false, adobe_none = false;
    int hmax = 0, vmax = 0;
    size_t pos = 2;
    // JPEG XT boxes (APP11 'JP'): the merging specification and the residual codestream, collected piece by piece
    struct XtBox {
        bool seen = false;
        int en = 0;
        uint64_t size = 0;
        std::vector<uint8_t> bytes;
    } xt_spec, xt_resi;
    bool xt_other = false;  // boxes this path does not cover (refinement data, alpha, curves, matrices, ...)

    for (;;) {
        // Behind the first scan the reference only warns about a missing EOI or bytes that are no marker and still delivers
        // the image (Frame::ParseTrailer marker/frame.cpp:1089-1110, Image::ParseTrailer codestream/image.cpp:1466-1486):
        // the end of the data is the end of the image, garbage is skipped up to the next 0xff.
        if (pos + 1 >= len) {
            if (!out.scans.empty()) break;
            FAIL(B200JPG_ERR_UNEXPECTED_EOF, "run out of data while looking for the next marker");
        }
        if (data[pos] != 0xff) {
            if (out.scans.empty()) FAIL(B200JPG_ERR_MALFORMED_STREAM, "expected a marker segment");
            const void *q = memchr(data + pos, 0xff, len - pos);
            pos = q ? (size_t)((const uint8_t *)q - data) : len;
            continue;
        }
        while (pos + 1 < len && data[pos + 1] == 0xff) pos++;  // filler, tables.cpp:1371-1373
        if (pos + 1 >= len) {
            if (!out.scans.empty()) break;
            FAIL(B200JPG_ERR_UNEXPECTED_EOF, "run out of data while looking for the next marker");
        }
        int m = data[pos + 1];
        pos += 2;
        if (m == 0xd9) break;  // EOI
        if (m >= 0xd0 && m <= 0xd7) continue;
        int seglen = c.u16(pos);
        if (seglen < 2 || pos + (size_t)seglen > len) FAIL(B200JPG_ERR_UNEXPECTED_EOF, "marker segment runs past the end of the stream");
        const uint8_t *s = data + pos + 2;
        int rem = seglen - 2;

        switch (m) {
        case 0xdb:  // DQT
            while (rem > 2) {
                int type = s[0] >> 4, target = s[0] & 15;
                s++, rem--;
                if (type > 1) FAIL(B200JPG_ERR_MALFORMED_STREAM, "DQT marker entry type must be either 0 or 1");
                if (target > 3) FAIL(B200JPG_ERR_MALFORMED_STREAM, "DQT marker target table must be between 0 and 3");
                int need = 64 * (type + 1);
                if (rem < need) FAIL(B200JPG_ERR_MALFORMED_STREAM, "DQT marker contains insufficient data");
                for (int i = 0; i < 64; i++) quant[target][i] = type ? (uint16_t)((s[2 * i] << 8) | s[2 * i + 1]) : s[i];
                quant_defined[target] = true;
                s += need, rem -= need;
            }
            if (rem != 0) FAIL(B200JPG_ERR_MALFORMED_STREAM, "DQT marker size corrupt");
            break;
        case 0xc4:  // DHT
            while (rem > 0) {
                int t = s[0];
                s++, rem--;
                if ((t >> 4) > 1) FAIL(B200JPG_ERR_MALFORMED_STREAM, "undefined Huffman table type");
                if ((t & 15) > 3) FAIL(B200JPG_ERR_MALFORMED_STREAM, "invalid Huffman table destination, must be between 0 and 3");
                if (rem < 16) FAIL(B200JPG_ERR_MALFORMED_STREAM, "Huffman table marker run out of data");
                int total = 0;
                for (int i = 0; i < 16; i++) total += s[i];
                if (rem < 16 + total) FAIL(B200JPG_ERR_MALFORMED_STREAM, "Huffman table marker run out of data");
                if (total > 256) FAIL(B200JPG_ERR_MALFORMED_STREAM, "Huffman table defines more than 256 symbols");
                HuffSpec &h = (t >> 4) ? ac[t & 3] : dc[t & 3];
                h.defined = true;
                memcpy(h.bits, s, 16);
                memcpy(h.vals, s + 16, (size_t)total);
                h.nvals = total;
                s += 16 + total, rem -= 16 + total;
            }
            break;
        case 0xdd:  // DRI
            if (seglen != 4) FAIL(B200JPG_ERR_MALFORMED_STREAM, "DRI restart interval definition marker size is invalid");
            dri = (uint32_t)c.u16(pos + 2);
            break;
        case 0xee:  // APP14: Adobe colour information (tables.cpp:2023-2025)
            if (rem >= 12 && memcmp(s, "Adobe", 5) == 0) {
                adobe_none = (s[11] == 0);
                if (out.scans.empty()) out.adobe_transform = s[11];  // libjpeg's examine_app14: the last one in front of the first scan
            }
            break;
        case 0xe1:  // APP1: Exif orientation, read in front of the first scan only (the reference skips the segment)
            if (out.scans.empty() && !exif_seen) {
                const int o = exif_orientation_of(s, (size_t)rem);
                if (o != 0) exif_seen = true, out.orientation = o;
            }
            break;
        case 0xeb:  // APP11: a piece of a JPEG XT box -- 'JP', enumerator, sequence number, LBox, TBox, payload (boxes/box.cpp:95-205)
            if (out.scans.empty() && rem >= 2 + 2 + 4 + 4 + 4 && s[0] == 'J' && s[1] == 'P') {
                const int en = (s[2] << 8) | s[3];
                const uint32_t lbox = ((uint32_t)s[8] << 24) | ((uint32_t)s[9] << 16) | ((uint32_t)s[10] << 8) | s[11];
                const uint32_t tbox = ((uint32_t)s[12] << 24) | ((uint32_t)s[13] << 16) | ((uint32_t)s[14] << 8) | s[15];
                const uint8_t *payload = s + 16;
                const size_t plen = (size_t)rem - 16;
                XtBox *box = nullptr;
                if (tbox == 0x53504543u) box = &xt_spec;       // 'SPEC'
                else if (tbox == 0x52455349u) box = &xt_resi;  // 'RESI'
                else if (tbox != 0x66747970u && tbox != 0x4c43484bu) xt_other = true;  // not 'ftyp', not 'LCHK' (checksum: not verified)
                if (box) {
                    if (lbox < 8) {  // 1 = XLBox, 0 = up to the end of the file
                        xt_other = true;
                    } else if (!box->seen) {
                        box->seen = true, box->en = en, box->size = lbox - 8;
                    } else if (box->en != en || box->size != lbox - 8) {
                        xt_other = true;  // a second box of the type
                        box = nullptr;
                    }
                    if (box && lbox >= 8) {
                        if (box->bytes.size() + plen > box->size)
                            FAIL(B200JPG_ERR_MALFORMED_STREAM, "more data in the application marker than indicated by the box contained within");
                        box->bytes.insert(box->bytes.end(), payload, payload + plen);
                    }
                }
            }
            break;
        case 0xc0:
        case 0xc1:
        case 0xc2: {
            if (have_sof) FAIL(B200JPG_ERR_MALFORMED_STREAM, "found a second frame header, hierarchical JPEG is not supported");
            if (seglen < 8) FAIL(B200JPG_ERR_MALFORMED_STREAM, "start of frame marker size invalid");
            fi.frame_type = (uint8_t)(m - 0xc0);
            fi.precision = s[0];
            if (m == 0xc0 && fi.precision != 8) FAIL(B200JPG_ERR_MALFORMED_STREAM, "frame precision in baseline mode must be 8");
            if (fi.precision != 8 && fi.precision != 12) FAIL(B200JPG_ERR_MALFORMED_STREAM, "frame precision in lossy mode must be 8 or 12");
            fi.height = (uint32_t)((s[1] << 8) | s[2]);
            fi.width = (uint32_t)((s[3] << 8) | s[4]);
            if (fi.width == 0) FAIL(B200JPG_ERR_MALFORMED_STREAM, "image width must not be zero");
            if (fi.height == 0) {
                // The height follows the first scan in a DNL marker (EntropyParser::ParseDNLMarker codestream/entropyparser.cpp:
                // 204-249, looked for in front of every MCU, entropyparser.hpp:147-152). The kernels want the geometry up front,
                // so the marker is looked up now: tables up to the first SOS, that scan's entropy coded segment, FF DC.
                size_t q = pos + (size_t)seglen;
                while (q + 3 < len && data[q] == 0xff && data[q + 1] != 0xda) {
                    if (data[q + 1] == 0xff) {
                        q++;
                        continue;
                    }
                    q += 2 + (size_t)c.u16(q + 2);
                }
                int hgt = -1;
                if (q + 3 < len && data[q] == 0xff && data[q + 1] == 0xda) {
                    std::vector<size_t> at;
                    std::vector<uint8_t> id;
                    const size_t e = index_ecs(c, q + 2 + (size_t)c.u16(q + 2), at, id);
                    if (e + 5 < len && data[e] == 0xff && data[e + 1] == 0xdc && c.u16(e + 2) == 4) hgt = c.u16(e + 4);
                }
                if (hgt <= 0) FAIL(B200JPG_ERR_MALFORMED_STREAM, "frame height is zero and no DNL marker follows the first scan");
                fi.height = (uint32_t)hgt;
            }
            int nc = s[5];
            if (nc < 1) FAIL(B200JPG_ERR_MALFORMED_STREAM, "number of components must be between 1 and 255");
            if (seglen - 8 != 3 * nc) FAIL(B200JPG_ERR_MALFORMED_STREAM, "frame header marker size is invalid");
            if (nc > B200JPG_MAX_COMPONENTS) FAIL(B200JPG_ERR_NOT_IMPLEMENTED, "more than four components are not supported by the GPU path");
            fi.ncomp = (uint8_t)nc;
            for (int i = 0; i < nc; i++) {
                fi.comp_id[i] = s[6 + 3 * i];
                fi.hs[i] = s[7 + 3 * i] >> 4;
                fi.vs[i] = s[7 + 3 * i] & 15;
                fi.tq[i] = s[8 + 3 * i];
                if (fi.hs[i] == 0 || fi.vs[i] == 0) FAIL(B200JPG_ERR_MALFORMED_STREAM, "frame marker corrupt, MCU size cannot be 0");
                if (fi.tq[i] > 3) FAIL(B200JPG_ERR_MALFORMED_STREAM, "quantization table identifier corrupt, must be >= 0 and <= 3");
                if (fi.hs[i] > hmax) hmax = fi.hs[i];
                if (fi.vs[i] > vmax) vmax = fi.vs[i];
            }
            fi.mcu_cols = (fi.width + 8 * hmax - 1) / (8 * hmax);
            fi.mcu_rows = (fi.height + 8 * vmax - 1) / (8 * vmax);
            fi.stored_blocks = 0;
            for (int i = 0; i < nc; i++) {
                if (hmax % fi.hs[i] || vmax % fi.vs[i])
                    FAIL(B200JPG_ERR_NOT_IMPLEMENTED, "subsampling factors are not integer, this is not supported");  // component.hpp:99-106
                fi.subx[i] = (uint8_t)(hmax / fi.hs[i]);
                fi.suby[i] = (uint8_t)(vmax / fi.vs[i]);
                fi.blocks_w[i] = fi.mcu_cols * fi.hs[i];
                fi.blocks_h[i] = fi.mcu_rows * fi.vs[i];
                uint32_t cw = (fi.width + fi.subx[i] - 1) / fi.subx[i], ch = (fi.height + fi.suby[i] - 1) / fi.suby[i];
                fi.stored_blocks += (uint64_t)((cw + 7) >> 3) * ((ch + 7) >> 3);
            }
            have_sof = true;
            break;
        }
        case 0xda: {
            if (!have_sof) FAIL(B200JPG_ERR_MALFORMED_STREAM, "found a start of scan before the frame header");
            if (out.scans.size() >= B200JPG_MAX_SCANS) FAIL(B200JPG_ERR_NOT_IMPLEMENTED, "too many scans for the GPU path");
            if (seglen < 8) FAIL(B200JPG_ERR_MALFORMED_STREAM, "marker length of the SOS marker invalid, must be at least 8 bytes long");
            ScanInfo sc;
            sc.ns = s[0];
            if (sc.ns < 1 || sc.ns > 4) FAIL(B200JPG_ERR_MALFORMED_STREAM, "number of components in scan is invalid, must be between 1 and 4");
            if (seglen != 2 * sc.ns + 6) FAIL(B200JPG_ERR_MALFORMED_STREAM, "length of the SOS marker is invalid");
            for (int i = 0; i < sc.ns; i++) {
                int id = s[1 + 2 * i], sel = s[2 + 2 * i], found = -1;
                for (int j = 0; j < fi.ncomp; j++)
                    if (fi.comp_id[j] == id) found = j;
                if (found < 0) FAIL(B200JPG_ERR_MALFORMED_STREAM, "SOS marker references a component that is not part of the frame");
                for (int j = 0; j < i; j++)
                    if (sc.comp[j] == found) FAIL(B200JPG_ERR_MALFORMED_STREAM, "SOS includes the same component twice");
                sc.comp[i] = found;
                sc.td[i] = sel >> 4;
                sc.ta[i] = sel & 15;
                if (sc.td[i] > 3) FAIL(B200JPG_ERR_MALFORMED_STREAM, "DC table index in SOS marker is out of range, must be at most 4");
                if (sc.ta[i] > 3) FAIL(B200JPG_ERR_MALFORMED_STREAM, "AC table index in SOS marker is out of range, must be at most 4");
            }
            // T.81 B.2.3 limits an interleaved MCU to ten blocks; the reference does not insist (its encoder writes 4x4 luma
            // sampling happily), so neither does this parser -- only the synchronisation path's per-MCU tables do (below)
            int blocks_per_mcu = 1;
            if (sc.ns > 1) {
                blocks_per_mcu = 0;
                for (int i = 0; i < sc.ns; i++) blocks_per_mcu += fi.hs[sc.comp[i]] * fi.vs[sc.comp[i]];
            }
            const uint8_t *t = s + 1 + 2 * sc.ns;
            sc.progressive = fi.frame_type == 2;
            sc.ss = t[0];
            sc.se = t[1];
            sc.ah = t[2] >> 4;
            sc.lowbit = t[2] & 15;
            if (sc.progressive) {  // marker/scan.cpp:257-302
                if (sc.ss > sc.se || sc.se > 63) FAIL(B200JPG_ERR_MALFORMED_STREAM, "spectral selection of the scan is invalid");
                if (sc.ss == 0 && sc.se != 0)
                    FAIL(B200JPG_ERR_MALFORMED_STREAM, "DC and AC coefficients must be coded in separate scans in the progressive mode");
                if (sc.ss != 0 && sc.ns != 1)
                    FAIL(B200JPG_ERR_MALFORMED_STREAM, "AC scans of the progressive mode must contain a single component");
                if (sc.ah != 0 && sc.ah != sc.lowbit + 1)
                    FAIL(B200JPG_ERR_MALFORMED_STREAM, "successive approximation must refine by one bit per scan");
            } else {
                if (sc.ss != 0 || sc.se != 63)
                    FAIL(B200JPG_ERR_MALFORMED_STREAM, "scan start must be zero and scan stop must be 63 for the sequential operating modes");
                if (sc.ah != 0)
                    FAIL(B200JPG_ERR_MALFORMED_STREAM, "successive approximation parameters must be zero for the sequential operating modes");
            }
            sc.dri = dri;
            sc.ecs_off = pos + (size_t)seglen;
            if (sc.ns > 1) {
                sc.mcu_cols = fi.mcu_cols;
                sc.mcu_rows = fi.mcu_rows;
            } else {  // sequentialscan.cpp:393-394: a single component scan walks that component's own block grid
                int ci = sc.comp[0];
                uint32_t cw = (fi.width + fi.subx[ci] - 1) / fi.subx[ci], ch = (fi.height + fi.suby[ci] - 1) / fi.suby[ci];
                sc.mcu_cols = (cw + 7) >> 3;
                sc.mcu_rows = (ch + 7) >> 3;
            }
            for (int i = 0; i < 4; i++) {
                sc.dc[i] = dc[i];
                sc.ac[i] = ac[i];
                memcpy(sc.quant[i], quant[i], sizeof(quant[i]));
                sc.quant_defined[i] = quant_defined[i];
            }
            for (int i = 0; i < sc.ns; i++) {
                const bool need_dc = !sc.progressive || (sc.ss == 0 && sc.ah == 0), need_ac = !sc.progressive || sc.se != 0;
                if ((need_dc && !dc[sc.td[i]].defined) || (need_ac && !ac[sc.ta[i]].defined))
                    FAIL(B200JPG_ERR_MALFORMED_STREAM, "Huffman decoder not specified for all components included in scan");  // sequentialscan.cpp:117-129
                if (!quant_defined[fi.tq[sc.comp[i]]])
                    FAIL(B200JPG_ERR_MALFORMED_STREAM, "quantization table for a component of the scan is not defined");
            }
            uint64_t total = (uint64_t)sc.mcu_cols * sc.mcu_rows;
            uint64_t per = sc.dri ? sc.dri : total;
            uint64_t nint = (total + per - 1) / per;
            // Untrusted header fields must not size allocations: every restart interval but the last is followed by a two
            // byte marker, so a stream of this length cannot hold more of them than that -- the rest would have to be
            // absent, which the reference turns into a failed resynchronisation or cleared MCUs. The index keeps at most
            // that many entries + 1; a frame that claims more is refused before anything is allocated.
            {
                const uint64_t room = (len - (pos + (size_t)seglen)) / 2 + 2;
                if (nint > room && nint > (1u << 16))
                    FAIL(B200JPG_ERR_MALFORMED_STREAM, "frame header promises more restart intervals than the stream can hold");
                if (total > (1ull << 31)) FAIL(B200JPG_ERR_NOT_IMPLEMENTED, "frame too large for the GPU path");
            }
            // A scan with restart markers that carries every component is the only scan of the frame: its entropy coded
            // segment runs up to the closing EOI, which is looked for from the end (bytes behind EOI are legal), and the
            // restart index is left to the device (restart_index_kernel) instead of a memchr pass over every byte here.
            if (device_index && !sc.progressive && sc.dri != 0 && sc.ns == (int)fi.ncomp) {
                size_t lo = (len > 4096) ? len - 4096 : 0, eoi = SIZE_MAX;
                if (lo < sc.ecs_off) lo = sc.ecs_off;
                for (size_t q = len; q >= lo + 2; q--)
                    if (data[q - 2] == 0xff && data[q - 1] == 0xd9) {
                        eoi = q - 2;
                        break;
                    }
                if (eoi != SIZE_MAX) {
                    sc.device_index = true;
                    sc.ecs_end = eoi;
                    sc.interval_off.assign((size_t)nint, sc.ecs_off);
                    sc.interval_end.assign((size_t)nint, eoi);
                    fi.n_intervals += (uint32_t)nint;
                    fi.ecs_bytes += sc.ecs_end - sc.ecs_off;
                    if (out.scans.empty()) fi.restart_interval = dri;
                    out.scans.push_back(std::move(sc));
                    goto parsed;  // nothing behind this scan is looked at
                }
            }
            // restart-interval index
            std::vector<size_t> rst_at;
            std::vector<uint8_t> rst_id;
            sc.ecs_end = index_ecs(c, sc.ecs_off, rst_at, rst_id);
            // The data ends inside the entropy coded segment (no marker follows). The reference's bit reader then hands out
            // zero bits without complaint (io/bitstream.cpp:103-105), so a cut inside the LAST interval still decodes; a cut
            // in front of a restart marker the scan needs makes ParseRestartMarker run out of data while resynchronising
            // (codestream/entropyparser.cpp:141-147): UNEXPECTED_EOF.
            sc.eof_tail = sc.ecs_end >= len;
            sc.interval_off.assign((size_t)nint, SIZE_MAX);
            sc.interval_end.assign((size_t)nint, sc.ecs_end);
            if (resolve_restart_sequence(rst_at, rst_id, sc.ecs_off, sc.ecs_end, sc.eof_tail, sc.interval_off, sc.interval_end) != 0)
                FAIL(B200JPG_ERR_UNEXPECTED_EOF, "run into end of file while trying to resync the entropy parser");
            // the data ends inside the scan's LAST interval: only then does the decoder read zero bits behind it
            sc.eof_tail = sc.eof_tail && sc.interval_off[nint - 1] != SIZE_MAX && sc.interval_end[nint - 1] >= len;
            // restart-less sequential scans of some size are cut up at synchronisation points on the device (specsync.hpp)
            sc.spec = !sc.progressive && nint == 1 && sc.ecs_end - sc.ecs_off >= kSpecMinBytes && blocks_per_mcu <= kSpecMaxBlocksPerMcu &&
                      getenv("B200JPG_NO_SPEC") == nullptr;
            fi.n_intervals += (uint32_t)nint;
            fi.ecs_bytes += sc.ecs_end - sc.ecs_off;
            if (out.scans.empty()) fi.restart_interval = dri;
            pos = sc.ecs_end;
            out.scans.push_back(std::move(sc));
            continue;
        }
        default:
            if (m == 0xc3 || (m >= 0xc5 && m <= 0xcf && m != 0xc8 && m != 0xcc))
                FAIL(B200JPG_ERR_NOT_IMPLEMENTED, "only baseline, extended sequential and progressive Huffman frames are supported by the GPU path");
            break;  // APPn, COM, JPG extensions: skipped by length (tables.cpp:1057-1072,1385-1399)
        }
        pos += (size_t)seglen;
    }
parsed:
    if (!have_sof) FAIL(B200JPG_ERR_MALFORMED_STREAM, "codestream contains no frame header");
    if (out.scans.empty()) FAIL(B200JPG_ERR_MALFORMED_STREAM, "codestream contains no scan");
    fi.nscans = (uint32_t)out.scans.size();
    fi.ycbcr = (fi.ncomp == 3 && !adobe_none) ? 1 : 0;  // tables.cpp:2023-2030
    if (xt_spec.seen || xt_resi.seen || xt_other) {
        // ---- JPEG XT: what of MergingSpecBox / ColorTransformerFactory::BuildColorTransformer (colortransformerfactory.cpp:
        // 217-300) this path covers
        int ocon = -1, ltrf = -1, rtrf = -1, ctrf = -1;
        if ((xt_spec.seen && xt_spec.bytes.size() != xt_spec.size) || (xt_resi.seen && xt_resi.bytes.size() != xt_resi.size))
            FAIL(B200JPG_ERR_MALFORMED_STREAM, "JPEG XT box is incomplete");
        const std::vector<uint8_t> &sp = xt_spec.bytes;
        size_t p = 0;
        while (p + 8 <= sp.size()) {  // the sub-boxes of the merging specification: LBox, TBox, payload
            const uint32_t lbox = ((uint32_t)sp[p] << 24) | ((uint32_t)sp[p + 1] << 16) | ((uint32_t)sp[p + 2] << 8) | sp[p + 3];
            const uint32_t tbox = ((uint32_t)sp[p + 4] << 24) | ((uint32_t)sp[p + 5] << 16) | ((uint32_t)sp[p + 6] << 8) | sp[p + 7];
            if (lbox < 8 || p + lbox > sp.size()) FAIL(B200JPG_ERR_MALFORMED_STREAM, "merging specification box is corrupt");
            if (tbox == 0x4f434f4eu && lbox == 11) ocon = sp[p + 8] | (sp[p + 9] << 8) | (sp[p + 10] << 16);  // 'OCON'
            else if (tbox == 0x4c545246u && lbox == 9) ltrf = sp[p + 8];                                       // 'LTRF'
            else if (tbox == 0x52545246u && lbox == 9) rtrf = sp[p + 8];                                       // 'RTRF'
            else if (tbox == 0x43545246u && lbox == 9) ctrf = sp[p + 8];                                       // 'CTRF'
            else xt_other = true;
            p += lbox;
        }
        if (p != sp.size()) FAIL(B200JPG_ERR_MALFORMED_STREAM, "merging specification box is corrupt");
        const char *nimpl = "JPEG XT profile outside the GPU path (covered: 8-bit base + 8-bit DCT residual, default tables, clamped output)";
        if (xt_other || !xt_spec.seen || fi.precision != 8 || (fi.ncomp != 1 && fi.ncomp != 3)) FAIL(B200JPG_ERR_NOT_IMPLEMENTED, nimpl);
        if (ocon != 0x02) FAIL(B200JPG_ERR_NOT_IMPLEMENTED, nimpl);                  // clamping only: no lossless, float, lookup, extra range bits
        if (ctrf != -1 && ctrf != (1 << 4)) FAIL(B200JPG_ERR_NOT_IMPLEMENTED, nimpl);  // C transformation: the identity
        if (fi.ncomp == 1) {
            if (ltrf != -1) FAIL(B200JPG_ERR_MALFORMED_STREAM, "Base transformation box exists even though the number of components is one");  // tables.cpp:2001-2003
            if (rtrf != -1 && rtrf != (1 << 4)) FAIL(B200JPG_ERR_NOT_IMPLEMENTED, nimpl);
        } else {
            if (ltrf == -1) out.xt.l_ycbcr = fi.ycbcr != 0;  // the JPEG default, tables.cpp:2023-2030
            else if (ltrf == (2 << 4)) out.xt.l_ycbcr = true;
            else if (ltrf == (1 << 4)) out.xt.l_ycbcr = false;
            else FAIL(B200JPG_ERR_NOT_IMPLEMENTED, nimpl);
            if (rtrf == -1 || rtrf == (2 << 4)) out.xt.r_ycbcr = true;  // tables.cpp:2052-2060
            else if (rtrf == (1 << 4)) out.xt.r_ycbcr = false;
            else FAIL(B200JPG_ERR_NOT_IMPLEMENTED, nimpl);  // RCT (lossless), free form
        }
        if (xt_resi.seen) {
            out.xt.present = true;
            out.xt.resi = std::move(xt_resi.bytes);
        } else {
            // a merging specification without a residual codestream (the reference encoder writes one into every grey file):
            // Extended | ClampFlag -- L transformation, identity tables, clamp (ycbcrtrafo.cpp:834-878 with rr = the DC shift):
            // the plain decode with the L transformation the box names
            if (fi.ncomp == 3) fi.ycbcr = out.xt.l_ycbcr ? 1 : 0;
        }
    }
    return B200JPG_OK;
}

int frame_colorspace(const ParsedFrame &pf) {
    const b200jpg_frame_info &fi = pf.info;
    if (fi.ncomp == 1) return B200JPG_COLORSPACE_GREY;
    if (fi.ncomp == 3) return fi.ycbcr ? B200JPG_COLORSPACE_YCBCR : B200JPG_COLORSPACE_RGB;
    if (fi.ncomp == 4 && fi.precision == 8 && pf.adobe_transform >= 0)
        return pf.adobe_transform == 0 ? B200JPG_COLORSPACE_CMYK : B200JPG_COLORSPACE_YCCK;
    return B200JPG_COLORSPACE_UNKNOWN;  // two components, an unmarked or a 12-bit four-component frame
}

uint32_t TableSet::lut_words() const {
    uint32_t v;
    memcpy(&v, blob.data() + 8, 4);
    return v;
}

int build_table_set(const ScanInfo &scan, TableSet &out, std::string &err) {
    // LUT entry layout: internal.hpp.  First level: top kLutL1Bits bits of the 16-bit window.
    std::vector<uint32_t> lut;
    uint16_t lut_off[8];
    const uint32_t kUnused = 0x80000000u | ((uint32_t)kQzBlockEnds << 19) | (31u << 5);
    const int L1 = kLutL1Bits, L2 = 16 - kLutL1Bits;
    // Progressive scans decode with the raw (run, size) of a symbol -- EOBn is a legal AC symbol there -- kept in [13:10]
    // and [4:0]; only the tables the scan kind reads are built.
    const bool need_dc = !scan.progressive || (scan.ss == 0 && scan.ah == 0), need_ac = !scan.progressive || scan.se != 0;
    for (int t = 0; t < 8; t++) {
        const HuffSpec &h = (t < 4) ? scan.dc[t] : scan.ac[t - 4];
        const bool is_ac = t >= 4;
        lut_off[t] = 0xffff;
        if (!h.defined || !(is_ac ? need_ac : need_dc)) continue;
        bool used = false;
        for (int i = 0; i < scan.ns; i++) used |= is_ac ? (scan.ta[i] == t - 4) : (scan.td[i] == t);
        if (!used) continue;
        size_t base = lut.size();
        if (base > 0xf000) FAIL(B200JPG_ERR_NOT_IMPLEMENTED, "Huffman tables too large for the GPU decoder tables");
        lut_off[t] = (uint16_t)base;
        lut.resize(base + ((size_t)1 << L1), kUnused);
        std::vector<int> sub_of((size_t)1 << L1, 0);
        int nsub = 0;
        uint32_t code = 0;  // left aligned in 16 bits (coding/huffmantemplate.cpp:823-826)
        int v = 0;
        for (int i = 0; i < 16; i++) {
            for (int j = 0; j < h.bits[i]; j++) {
                if (v >= h.nvals) FAIL(B200JPG_ERR_MALFORMED_STREAM, "Huffman table marker depends on undefined data");
                const uint8_t sym = h.vals[v++];
                const uint32_t last = code + (1u << (15 - i));
                if (last > 0x10000u)
                    FAIL(B200JPG_ERR_MALFORMED_STREAM, "Huffman table corrupt - entry depends on more bits than available for the bit length");
                const uint32_t len = (uint32_t)i + 1;
                uint32_t s, r, bad = 0;
                if (is_ac) {
                    s = sym & 15u;
                    r = sym >> 4;
                    if (s == 0 && r != 0 && r != 15 && !scan.progressive) bad = 1;  // sequentialscan.cpp:750-752: not a baseline symbol
                } else {
                    s = sym;
                    r = 0;
                    if (sym > 15) {  // sequentialscan.cpp:688-690
                        bad = 1;
                        s = 0;
                    }
                }
                uint32_t step = 0;
                if (is_ac) step = bad ? (uint32_t)kQzBlockEnds : (s != 0 ? r + 1u : (r == 15 ? 16u : (uint32_t)kQzBlockEnds));
                uint32_t entry = (bad << 31) | ((len + s) << 26) | (step << 19) | (len << 5) | s;
                if (scan.progressive) entry = (bad << 31) | ((len + s) << 26) | (r << 10) | (len << 5) | s;
                if ((int)len <= L1) {
                    for (uint32_t q = code >> L2, qlast = last >> L2; q < qlast; q++) lut[base + q] = entry;
                } else {
                    for (uint32_t c16 = code; c16 < last; c16++) {
                        const uint32_t q = c16 >> L2;
                        if (!sub_of[q]) {
                            sub_of[q] = ++nsub;
                            if (nsub > 255) FAIL(B200JPG_ERR_NOT_IMPLEMENTED, "Huffman tables too large for the GPU decoder tables");
                            lut.resize(base + ((size_t)1 << L1) + ((size_t)nsub << L2), kUnused);
                            lut[base + q] = (uint32_t)(sub_of[q] - 1) << 10;  // len field 0 -> second level
                        }
                        lut[base + ((size_t)1 << L1) + ((size_t)(sub_of[q] - 1) << L2) + (c16 & ((1u << L2) - 1))] = entry;
                    }
                }
                code = last;
            }
        }
    }
    if (lut.size() > 0xffffu) FAIL(B200JPG_ERR_NOT_IMPLEMENTED, "Huffman tables too large for the GPU decoder tables");
    // quantisation + de-zigzag: per table kQzEntries (q, byte offset) pairs indexed by the zig-zag position k. 64..95 is
    // the "AC coefficient decoding out of sync" case of sequentialscan.cpp:764-766 (flagged); 96.. is where symbols that
    // end the block point (EOB, error entries): a zero parked in the pad slot, like the flagged ones
    size_t total = kTableHeaderBytes + lut.size() * 4;
    total = (total + 15) & ~(size_t)15;
    out.blob.assign(total, 0);
    uint32_t hdr[4] = {kTableMagic, (uint32_t)total, (uint32_t)lut.size(), scan.progressive ? 1u : 0u};
    memcpy(out.blob.data(), hdr, 16);
    memcpy(out.blob.data() + 16, lut_off, 16);
    uint32_t *qz = (uint32_t *)(out.blob.data() + 32);
    for (int t = 0; t < 4; t++)
        for (int k = 0; k < kQzEntries; k++) {
            uint32_t q, off;
            if (k < 64) {
                uint32_t delta = scan.quant_defined[t] ? scan.quant[t][k] : 0;
                if (((uint64_t)delta << scan.lowbit) >= (1u << 24))
                    FAIL(B200JPG_ERR_NOT_IMPLEMENTED, "quantisation step times point transform too large for the GPU path");
                q = delta << scan.lowbit;
                off = 2u * kZigZagToRaster[k];
            } else {
                // 64..95: a coefficient whose run left the block (sequentialscan.cpp:764-766). The multiplier 2^16 turns any
                // non-zero amplitude into a product beyond the int16 store -- reported as MALFORMED_STREAM like a genuine
                // overflow --, while a ZRL that steps over position 63 lands here with amplitude 0 and ends the block
                // silently, as in the reference (:717-719)
                q = (k < kQzBlockEnds) ? 0x00010000u : 0u;
                off = 128;  // first pad halfword of the lane's staging block
            }
            qz[(t * kQzEntries + k) * 2] = q;
            qz[(t * kQzEntries + k) * 2 + 1] = off;
        }
    memcpy(out.blob.data() + kTableHeaderBytes, lut.data(), lut.size() * 4);
    return B200JPG_OK;
}

}  // namespace b200jpg
