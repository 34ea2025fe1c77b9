/*
 * oracle/jpeg_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE (see jpeg_oracle.h).
 *
 * CPU restatement, in plain C99, of the reference's sequential-Huffman JPEG decode path.  It is written
 * from the behaviour of the reference (thorfdbg/libjpeg, /root/reference), each function citing the
 * file:line it follows; it is not a copy of that code (the reference is C++ objects over hook-backed
 * streams and per-line linked lists; this is flat arrays over one in-memory byte view).
 *
 * Scope: SOF0 / 8-bit SOF1 frames, 1..4 components, sampling factors whose ratios to the maximum are 1 or 2
 * (so 4:4:4, 4:2:2, 4:4:0, 4:2:0), interleaved or non-interleaved sequential scans, DRI, byte stuffing.
 * Arithmetic widths follow the reference: int32 ("LONG") in the IDCT and the upsampler, int64 ("QUAD")
 * products in the colour transform.
 */
#include "jpeg_oracle.h"

#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------------ */
/* zig-zag index -> raster position x + 8*y.  Follows dct/dct.cpp:57-73 (DCT::ScanOrder).            */
const int jpgo_scan_order[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

/* ------------------------------------------------------------------------------------------------ */
/* Huffman tables: DHT payload kept as BITS/HUFFVAL (coding/huffmantemplate.cpp:878-904), decoder
 * built as the reference's two-level 8+8 bit lookup (coding/huffmantemplate.cpp:802-874).            */
typedef struct {
    int defined;
    uint8_t bits[16];
    uint8_t vals[256];
    int nvals;
    uint8_t sym1[256], len1[256]; /* len1: 1..8 direct, 0 = use second level, 0xff = unused           */
    uint8_t has2[256];
    uint8_t *sym2, *len2;         /* [256][256], rows valid where has2[msb]                            */
} hufftab;

int jpgo_build_huffman(const uint8_t bits[16], const uint8_t *vals, int nvals, uint8_t sym1[256],
                       uint8_t len1[256], uint8_t *sym2, uint8_t *len2, uint8_t has2[256]) {
    uint32_t code = 0; /* left-aligned in 16 bits, huffmantemplate.cpp:823-826 */
    int i, j, v = 0;
    memset(len1, 0xff, 256); /* huffmandecoder.hpp:87 */
    memset(sym1, 0, 256);
    memset(has2, 0, 256);
    for (i = 0; i < 16; i++) {
        for (j = 0; j < bits[i]; j++) {
            uint8_t symbol;
            uint32_t last, q, qlast;
            if (v >= nvals) return JPGO_ERR_MALFORMED_STREAM; /* :819-820 */
            symbol = vals[v++];
            last = code + (1u << (15 - i));
            if (last > 0x10000u) return JPGO_ERR_MALFORMED_STREAM; /* :829-831 */
            q = code >> 8;
            qlast = last >> 8;
            if (i < 8) { /* code of <= 8 bits fills whole first-level slots, :837-845 */
                do {
                    sym1[q] = symbol;
                    len1[q] = (uint8_t)(i + 1);
                } while (++q < qlast);
                code = last;
            } else { /* long code: first level says "second level", :846-862 */
                if (!has2[q]) {
                    has2[q] = 1;
                    memset(len2 + 256 * q, 0xff, 256);
                    memset(sym2 + 256 * q, 0, 256);
                }
                sym1[q] = symbol;
                len1[q] = 0;
                do {
                    sym2[256 * q + (code & 0xff)] = symbol;
                    len2[256 * q + (code & 0xff)] = (uint8_t)(i + 1);
                } while (++code < last);
            }
        }
    }
    return JPGO_OK;
}

/* ------------------------------------------------------------------------------------------------ */
/* Bit reader.  Follows io/bitstream.hpp:106-208 and io/bitstream.cpp:56-138: a 32-bit MSB-first window
 * refilled bytewise while it holds <= 24 bits; FF00 -> FF; FF xx (xx != 0) is a marker: stop there,
 * do not consume it and hand out eight zero bits per Fill() call; end of data likewise; an error is
 * raised only when a request is larger than the (possibly zero-padded) window after one Fill().      */
typedef struct {
    const uint8_t *p, *end;
    uint32_t b;
    int bits;
    int marker, eof;
    int error;
} bitreader;

static void br_open(bitreader *br, const uint8_t *p, const uint8_t *end) {
    br->p = p;
    br->end = end;
    br->b = 0;
    br->bits = 0;
    br->marker = br->eof = 0;
    br->error = 0;
}

static void br_fill(bitreader *br) {
    do {
        if (br->p >= br->end) { /* bitstream.cpp:103-105: EOF adds 8 zero bits and keeps looping */
            br->eof = 1;
            br->bits += 8;
        } else if (br->p[0] == 0xff) {
            if (br->p + 1 < br->end && br->p[1] == 0x00) { /* :87-95 */
                br->b |= (uint32_t)0xff << (24 - br->bits);
                br->bits += 8;
                br->p += 2;
            } else { /* :96-101 marker (or FF at the very end of the data) */
                br->marker = 1;
                br->bits += 8;
                break;
            }
        } else {
            br->b |= (uint32_t)br->p[0] << (24 - br->bits);
            br->bits += 8;
            br->p++;
        }
    } while (br->bits <= 24);
}

static void br_report(bitreader *br) { /* bitstream.cpp:125-138 */
    if (br->error) return;
    br->error = (br->eof || br->marker) ? JPGO_ERR_UNEXPECTED_EOF : JPGO_ERR_MALFORMED_STREAM;
}

static uint32_t br_get(bitreader *br, int n) { /* bitstream.hpp:168-186 */
    uint32_t v;
    if (n > br->bits) {
        br_fill(br);
        if (n > br->bits) {
            br_report(br);
            return 0;
        }
    }
    v = br->b >> (32 - n);
    br->b <<= n;
    br->bits -= n;
    return v;
}

static uint32_t br_peekword(bitreader *br) { /* bitstream.hpp:191-197 */
    if (br->bits < 16) br_fill(br);
    return br->b >> 16;
}

static void br_skip(bitreader *br, int n) { /* bitstream.hpp:201-208 */
    if (n > br->bits) {
        br_report(br);
        return;
    }
    br->b = (n >= 32) ? 0 : (br->b << n);
    br->bits -= n;
}

static int huff_get(const hufftab *t, bitreader *br) { /* coding/huffmandecoder.hpp:103-124 */
    uint32_t data = br_peekword(br);
    uint32_t msb = data >> 8;
    int symbol, size;
    if (t->len1[msb]) {
        symbol = t->sym1[msb];
        size = t->len1[msb];
    } else {
        symbol = t->sym2[256 * msb + (data & 0xff)];
        size = t->len2[256 * msb + (data & 0xff)];
    }
    br_skip(br, size); /* size 0xff on unused entries -> error */
    return symbol;
}

/* ------------------------------------------------------------------------------------------------ */
/* One block.  Follows codestream/sequentialscan.cpp:678-773 for the sequential (non-progressive,
 * non-residual, no large-range) case; lowbit is the point transform of the SOS (scan.cpp:257).       */
static void decode_block(int32_t *block, const hufftab *dc, const hufftab *ac, int32_t *prevdc, int lowbit,
                         bitreader *br) {
    int32_t diff = 0;
    int value = huff_get(dc, br);
    int k;
    if (br->error) return;
    if (value > 0) {
        int32_t v = (int32_t)1 << (value - 1);
        if (value > 15) { /* :688-690 */
            br->error = JPGO_ERR_MALFORMED_STREAM;
            return;
        }
        diff = (int32_t)br_get(br, value);
        if (br->error) return;
        if (diff < v) diff += (int32_t)(-(1 << value)) + 1;
    }
    *prevdc += diff;
    block[0] = (int32_t)((uint32_t)*prevdc << lowbit);

    k = 1;
    do {
        int rs = huff_get(ac, br);
        int r = rs >> 4, s = rs & 15;
        int32_t v, d;
        if (br->error) return;
        if (s == 0) {
            if (r == 15) { /* ZRL: `continue` re-tests k <= 63, :717-719 */
                k += 16;
                continue;
            }
            if (r == 0) break; /* EOB, :722-726 with skip = 0 */
            br->error = JPGO_ERR_MALFORMED_STREAM; /* :750-752 */
            return;
        }
        v = (int32_t)1 << (s - 1);
        k += r;
        d = (int32_t)br_get(br, s);
        if (br->error) return;
        if (d < v) d += (int32_t)(-(1 << s)) + 1;
        if (k >= 64) { /* :764-766 */
            br->error = JPGO_ERR_MALFORMED_STREAM;
            return;
        }
        block[jpgo_scan_order[k]] = (int32_t)((uint32_t)d << lowbit);
        k++;
    } while (k <= 63);
}

/* ------------------------------------------------------------------------------------------------ */
/* Progressive scans.  First passes: codestream/sequentialscan.cpp:678-773 with m_bProgressive (EOB runs
 * :722-726, point transform `<< lowbit`); refinement passes: codestream/refinementscan.cpp:584-690.
 * `skip` is the number of blocks an EOB run still covers (reset by Restart()).                        */
static void decode_block_first(int32_t *block, const hufftab *dc, const hufftab *ac, int32_t *prevdc, const jpgo_scan *sc,
                               unsigned *skip, bitreader *br) {
    if (sc->ss == 0) { /* DC, first pass: like the sequential case, :682-701 */
        int32_t diff = 0;
        int value = huff_get(dc, br);
        if (br->error) return;
        if (value > 0) {
            if (value > 15) {
                br->error = JPGO_ERR_MALFORMED_STREAM;
                return;
            }
            diff = (int32_t)br_get(br, value);
            if (br->error) return;
            if (diff < ((int32_t)1 << (value - 1))) diff += (int32_t)(-(1 << value)) + 1;
        }
        *prevdc += diff;
        block[0] = (int32_t)((uint32_t)*prevdc << sc->al);
    }
    if (sc->se) { /* AC, first pass */
        int k = sc->ss;
        if (*skip > 0) { /* inside an EOB run: the block stays as it is */
            (*skip)--;
            return;
        }
        do {
            int rs = huff_get(ac, br);
            int r = rs >> 4, s = rs & 15;
            int32_t d;
            if (br->error) return;
            if (s == 0) {
                if (r == 15) { /* ZRL; `continue` re-tests k <= Se */
                    k += 16;
                    continue;
                }
                *skip = 1u << r; /* EOBn: this block and 2^r + extra - 1 more */
                if (r) *skip |= br_get(br, r);
                (*skip)--;
                return;
            }
            k += r;
            d = (int32_t)br_get(br, s);
            if (br->error) return;
            if (d < ((int32_t)1 << (s - 1))) d += (int32_t)(-(1 << s)) + 1;
            if (k >= 64) { /* the reference tests against 64, not against Se */
                br->error = JPGO_ERR_MALFORMED_STREAM;
                return;
            }
            block[jpgo_scan_order[k]] = (int32_t)((uint32_t)d << sc->al);
            k++;
        } while (k <= sc->se);
    }
}

static void correct(int32_t *c, int al, bitreader *br) { /* one correction bit, away from zero (:616-626) */
    if (br_get(br, 1)) *c += (*c > 0) ? ((int32_t)1 << al) : -((int32_t)1 << al);
}

static void decode_block_refine(int32_t *block, const hufftab *ac, const jpgo_scan *sc, unsigned *skip, bitreader *br) {
    if (sc->ss == 0) { /* DC refinement: one raw bit, :588-592 */
        block[0] |= (int32_t)br_get(br, 1) << sc->al;
        return;
    }
    {
        int k = sc->ss;
        if (*skip == 0) {
            while (k <= sc->se) {
                int rs = huff_get(ac, br);
                int r = rs >> 4, s = rs & 15;
                int32_t val = 0;
                if (br->error) return;
                if (s == 0) {
                    if (r != 15) { /* EOBn: the rest of this block (and of the run) only takes correction bits */
                        *skip = 1u << r;
                        if (r) *skip |= br_get(br, r);
                        break;
                    }
                    /* ZRL: sixteen zero-valued positions */
                } else if (s != 1) { /* the reference warns and keeps going with a zero amplitude, :659-668 */
                    r = 0;
                } else {
                    val = br_get(br, 1) ? ((int32_t)1 << sc->al) : -((int32_t)1 << sc->al);
                }
                /* pass r zero-valued coefficients; the significant ones on the way take their correction bit */
                while (k <= sc->se) {
                    int32_t *c = &block[jpgo_scan_order[k]];
                    if (*c) {
                        correct(c, sc->al, br);
                    } else {
                        if (r == 0) break;
                        r--;
                    }
                    k++;
                }
                if (br->error) return;
                if (k <= sc->se) block[jpgo_scan_order[k]] = val; /* the zero-valued position that ends the run */
                k++;
            }
        }
        if (*skip > 0) {
            for (; k <= sc->se; k++) {
                int32_t *c = &block[jpgo_scan_order[k]];
                if (*c) correct(c, sc->al, br);
            }
            (*skip)--;
        }
    }
}

/* ------------------------------------------------------------------------------------------------ */
/* marker parser                                                                                       */
typedef struct {
    hufftab dc[4], ac[4];
    int lowbit[JPGO_MAX_SCANS];
    /* snapshot of which DHT slots each scan uses is taken at decode time by re-walking the stream */
} decoder_tables;

static int rd16(const uint8_t *d, size_t n, size_t pos) {
    if (pos + 1 >= n) return -1;
    return (d[pos] << 8) | d[pos + 1];
}

/* Find the end of an entropy coded segment: offset of the first FF xx with xx not in {00, FF, D0..D7}.
 * (the bit reader stops at any marker, io/bitstream.cpp:96-101; RSTn are consumed by
 * EntropyParser::ParseRestartMarker, codestream/entropyparser.cpp:117-136)                           */
static size_t find_ecs_end(const uint8_t *d, size_t n, size_t pos) {
    while (pos < n) {
        const uint8_t *q = (const uint8_t *)memchr(d + pos, 0xff, n - pos);
        if (!q) return n;
        pos = (size_t)(q - d);
        if (pos + 1 >= n) return n;
        if (d[pos + 1] == 0x00 || (d[pos + 1] >= 0xd0 && d[pos + 1] <= 0xd7)) {
            pos += 2;
        } else if (d[pos + 1] == 0xff) {
            pos += 1;
        } else {
            return pos;
        }
    }
    return n;
}

typedef void (*dht_cb)(void *user, int slot_is_ac, int th, const uint8_t *bits, const uint8_t *vals, int nvals);

/* Walks the marker segments.  Follows codestream/decoder.cpp:77, codestream/tables.cpp:1003-1420
 * (DQT/DHT/DRI/APPn/COM), marker/frame.cpp:111-214 (SOF), marker/scan.cpp:163-315 (SOS).
 * When `tabs` is non-NULL the Huffman tables in effect at scan `want_scan` are captured.
 * When `latched` is non-NULL it receives the quantiser of every component (raster order): its slot's table as it stood at
 * the first scan that holds the component -- the reference builds the component's IDCT there (BlockBuffer::
 * ResetToStartOfScan control/blockbuffer.cpp:185-197) and a later DQT does not reach it; a component no scan holds takes
 * the slot's last definition.                                                                          */
static int walk(const uint8_t *d, size_t n, jpgo_info *info, decoder_tables *tabs, int want_scan, uint16_t (*latched)[64]) {
    size_t pos = 2;
    int have_sof = 0, dri = 0, adobe_none = 0, seen = 0, i;
    if (n < 4 || d[0] != 0xff || d[1] != 0xd8) return JPGO_ERR_MALFORMED_STREAM; /* no SOI */
    memset(info, 0, sizeof(*info));
    for (;;) {
        int m, len;
        /* Behind the first scan the reference only WARNS about a missing EOI or out-of-sync bytes and delivers the
         * image (Frame::ParseTrailer marker/frame.cpp:1089-1110, Image::ParseTrailer codestream/image.cpp:1466-1486):
         * end of data = end of image, garbage is skipped up to the next 0xff. */
        if (pos + 1 >= n) {
            if (info->nscans > 0) break;
            return JPGO_ERR_UNEXPECTED_EOF;
        }
        if (d[pos] != 0xff) {
            if (info->nscans == 0) return JPGO_ERR_MALFORMED_STREAM;
            while (pos < n && d[pos] != 0xff) pos++;
            continue;
        }
        while (pos + 1 < n && d[pos + 1] == 0xff) pos++; /* filler bytes, tables.cpp:1371-1373 */
        if (pos + 1 >= n) {
            if (info->nscans > 0) break;
            return JPGO_ERR_UNEXPECTED_EOF;
        }
        m = d[pos + 1];
        pos += 2;
        if (m == 0xd9) break; /* EOI */
        if (m >= 0xd0 && m <= 0xd7) continue; /* stray RSTn between segments */
        len = rd16(d, n, pos);
        if (len < 2 || pos + (size_t)len > n) return JPGO_ERR_UNEXPECTED_EOF;
        switch (m) {
        case 0xdb: { /* DQT, marker/quantization.cpp:474-537 */
            size_t p = pos + 2;
            int rem = len - 2;
            while (rem > 2) {
                int type = d[p] >> 4, target = d[p] & 15;
                p++;
                rem--;
                if (type > 1 || target > 3) return JPGO_ERR_MALFORMED_STREAM;
                if (rem < 64 * (type + 1)) return JPGO_ERR_MALFORMED_STREAM;
                for (i = 0; i < 64; i++) {
                    int v = type ? ((d[p] << 8) | d[p + 1]) : d[p];
                    p += type + 1;
                    info->quant[target][jpgo_scan_order[i]] = (uint16_t)v; /* zig-zag -> raster */
                }
                rem -= 64 * (type + 1);
                info->quant_defined[target] = 1;
            }
            if (rem != 0) return JPGO_ERR_MALFORMED_STREAM;
            break;
        }
        case 0xc4: { /* DHT, marker/huffmantable.cpp:127-169 + coding/huffmantemplate.cpp:878-904 */
            size_t p = pos + 2;
            int rem = len - 2;
            while (rem > 0) {
                int t = d[p], tc = t >> 4, th = t & 15, total = 0;
                p++;
                rem--;
                if (tc > 1 || th > 3) return JPGO_ERR_MALFORMED_STREAM;
                if (rem < 16) return JPGO_ERR_MALFORMED_STREAM;
                for (i = 0; i < 16; i++) total += d[p + i];
                if (rem < 16 + total || total > 256) return JPGO_ERR_MALFORMED_STREAM;
                if (tabs) {
                    hufftab *h = tc ? &tabs->ac[th] : &tabs->dc[th];
                    h->defined = 1;
                    memcpy(h->bits, d + p, 16);
                    memcpy(h->vals, d + p + 16, (size_t)total);
                    h->nvals = total;
                }
                p += 16 + (size_t)total;
                rem -= 16 + total;
            }
            break;
        }
        case 0xdd: /* DRI, marker/restartintervalmarker.cpp:80-102 (16-bit for JPEG) */
            if (len != 4) return JPGO_ERR_MALFORMED_STREAM;
            dri = rd16(d, n, pos + 2);
            break;
        case 0xee: /* APP14 Adobe: colour transform flag 0 = none, marker/adobemarker.cpp */
            if (len >= 14 && memcmp(d + pos + 2, "Adobe", 5) == 0) adobe_none = (d[pos + 13] == 0);
            break;
        case 0xc0:
        case 0xc1:
        case 0xc2: { /* SOF0 / SOF1, marker/frame.cpp:111-214, marker/component.cpp:86-111 */
            size_t p = pos + 2;
            if (have_sof) return JPGO_ERR_MALFORMED_STREAM;
            if (len < 8) return JPGO_ERR_MALFORMED_STREAM;
            info->frame_type = m - 0xc0;
            info->precision = d[p];
            if (m == 0xc0 && info->precision != 8) return JPGO_ERR_MALFORMED_STREAM; /* frame.cpp: baseline is 8 bit */
            if (info->precision != 8 && info->precision != 12) return JPGO_ERR_NOT_IMPLEMENTED; /* lossy modes: 8 or 12 */
            info->height = rd16(d, n, p + 1);
            info->width = rd16(d, n, p + 3);
            info->ncomp = d[p + 5];
            if (info->width == 0) return JPGO_ERR_MALFORMED_STREAM;
            if (info->height == 0) { /* the height follows the first scan in a DNL marker (entropyparser.cpp:204-249, entropyparser.hpp:147-152) */
                size_t q = pos + (size_t)len, e;
                int hgt = -1;
                while (q + 3 < n && d[q] == 0xff && d[q + 1] != 0xda) { /* tables up to the first SOS */
                    if (d[q + 1] == 0xff) {
                        q++;
                        continue;
                    }
                    q += 2 + (size_t)rd16(d, n, q + 2);
                }
                if (q + 3 < n && d[q + 1] == 0xda) {
                    e = find_ecs_end(d, n, q + 2 + (size_t)rd16(d, n, q + 2));
                    if (e + 5 < n && d[e] == 0xff && d[e + 1] == 0xdc && rd16(d, n, e + 2) == 4) hgt = rd16(d, n, e + 4);
                }
                if (hgt <= 0) return JPGO_ERR_MALFORMED_STREAM;
                info->height = hgt;
            }
            if (info->ncomp < 1) return JPGO_ERR_MALFORMED_STREAM;
            if (info->ncomp > JPGO_MAX_COMP) return JPGO_ERR_NOT_IMPLEMENTED;
            if (len - 8 != 3 * info->ncomp) return JPGO_ERR_MALFORMED_STREAM;
            for (i = 0; i < info->ncomp; i++) {
                info->cid[i] = d[p + 6 + 3 * i];
                info->hs[i] = d[p + 7 + 3 * i] >> 4;
                info->vs[i] = d[p + 7 + 3 * i] & 15;
                info->tq[i] = d[p + 8 + 3 * i];
                if (info->hs[i] == 0 || info->vs[i] == 0 || info->tq[i] > 3) return JPGO_ERR_MALFORMED_STREAM;
                if (info->hs[i] > info->hmax) info->hmax = info->hs[i];
                if (info->vs[i] > info->vmax) info->vmax = info->vs[i];
            }
            info->mcu_cols = (info->width + 8 * info->hmax - 1) / (8 * info->hmax);
            info->mcu_rows = (info->height + 8 * info->vmax - 1) / (8 * info->vmax);
            for (i = 0; i < info->ncomp; i++) {
                int cw, ch;
                if (info->hmax % info->hs[i] || info->vmax % info->vs[i])
                    return JPGO_ERR_NOT_IMPLEMENTED; /* marker/component.hpp:99-106 */
                info->subx[i] = info->hmax / info->hs[i];
                info->suby[i] = info->vmax / info->vs[i];
                if (info->subx[i] > 4 || info->suby[i] > 4) return JPGO_ERR_NOT_IMPLEMENTED; /* upsamplerbase.cpp:335-404 */
                info->bw[i] = info->mcu_cols * info->hs[i];
                info->bh[i] = info->mcu_rows * info->vs[i];
                cw = (info->width + info->subx[i] - 1) / info->subx[i];
                ch = (info->height + info->suby[i] - 1) / info->suby[i];
                info->sbw[i] = (cw + 7) >> 3;
                info->sbh[i] = (ch + 7) >> 3;
            }
            have_sof = 1;
            break;
        }
        case 0xda: { /* SOS, marker/scan.cpp:163-315 */
            size_t p = pos + 2;
            jpgo_scan *sc;
            int ns, j;
            if (!have_sof) return JPGO_ERR_MALFORMED_STREAM;
            if (info->nscans >= JPGO_MAX_SCANS) return JPGO_ERR_NOT_IMPLEMENTED;
            sc = &info->scan[info->nscans];
            if (len < 8) return JPGO_ERR_MALFORMED_STREAM;
            ns = d[p];
            if (ns < 1 || ns > 4 || len != 2 * ns + 6) return JPGO_ERR_MALFORMED_STREAM;
            sc->ns = ns;
            for (i = 0; i < ns; i++) {
                int id = d[p + 1 + 2 * i], sel = d[p + 2 + 2 * i], found = -1;
                for (j = 0; j < info->ncomp; j++)
                    if (info->cid[j] == id) found = j;
                if (found < 0) return JPGO_ERR_MALFORMED_STREAM;
                for (j = 0; j < i; j++)
                    if (sc->comp[j] == found) return JPGO_ERR_MALFORMED_STREAM;
                sc->comp[i] = found;
                if (!(seen & (1 << found)) && info->quant_defined[info->tq[found]]) {
                    if (latched) memcpy(latched[found], info->quant[info->tq[found]], sizeof(latched[found]));
                    seen |= 1 << found;
                }
                sc->td[i] = sel >> 4;
                sc->ta[i] = sel & 15;
                if (sc->td[i] > 3 || sc->ta[i] > 3) return JPGO_ERR_MALFORMED_STREAM;
            }
            sc->ss = d[p + 1 + 2 * ns];
            sc->se = d[p + 2 + 2 * ns];
            sc->ah = d[p + 3 + 2 * ns] >> 4;
            sc->al = d[p + 3 + 2 * ns] & 15;
            if (info->frame_type == 2) { /* marker/scan.cpp:257-302 */
                if (sc->ss > sc->se || sc->se > 63) return JPGO_ERR_MALFORMED_STREAM;
                if (sc->ss == 0 && sc->se != 0) return JPGO_ERR_MALFORMED_STREAM; /* DC and AC must be coded separately */
                if (sc->ss != 0 && ns != 1) return JPGO_ERR_MALFORMED_STREAM;       /* AC scans carry one component */
                if (sc->ah != 0 && sc->ah != sc->al + 1) return JPGO_ERR_MALFORMED_STREAM; /* one bit per refinement */
            } else {
                if (sc->ss != 0 || sc->se != 63) return JPGO_ERR_MALFORMED_STREAM; /* :273-276 */
                if (sc->ah != 0) return JPGO_ERR_MALFORMED_STREAM;                  /* :280-282 */
            }
            if (tabs) tabs->lowbit[info->nscans] = sc->al;
            sc->restart_interval = dri;
            sc->ecs_offset = pos + (size_t)len;
            sc->ecs_end = find_ecs_end(d, n, sc->ecs_offset);
            if (ns > 1) {
                sc->mcu_cols = info->mcu_cols;
                sc->mcu_rows = info->mcu_rows;
            } else { /* single component scan: MCU = one block over the component's own grid */
                sc->mcu_cols = info->sbw[sc->comp[0]];
                sc->mcu_rows = info->sbh[sc->comp[0]];
            }
            info->nscans++;
            if (tabs && info->nscans - 1 == want_scan) {
                info->ycbcr = (info->ncomp == 3 && !adobe_none);
                return JPGO_OK; /* tables captured as of this scan */
            }
            pos = sc->ecs_end;
            continue;
        }
        default:
            if (m == 0xc3 || (m >= 0xc5 && m <= 0xcf && m != 0xc8 && m != 0xcc))
                return JPGO_ERR_NOT_IMPLEMENTED; /* lossless / arithmetic / hierarchical */
            break; /* APPn, COM, everything else: skipped by length (tables.cpp:1057-1072,1385-1399) */
        }
        pos += (size_t)len;
    }
    if (!have_sof || info->nscans == 0) return JPGO_ERR_MALFORMED_STREAM;
    for (i = 0; latched && i < info->ncomp; i++)
        if (!(seen & (1 << i))) memcpy(latched[i], info->quant[info->tq[i]], sizeof(latched[i]));
    info->ycbcr = (info->ncomp == 3 && !adobe_none); /* tables.cpp:2023-2030 */
    return JPGO_OK;
}

int jpgo_read_info(const uint8_t *data, size_t len, jpgo_info *info) { return walk(data, len, info, NULL, -1, NULL); }

/* `info` of the stream rewritten for reconstruction: component c dequantises through slot c, which holds the quantiser it
 * latched (walk) */
static int latched_quantisers(const uint8_t *data, size_t len, jpgo_info *info) {
    uint16_t q[JPGO_MAX_COMP][64];
    int defined[JPGO_MAX_COMP], c, rc;
    jpgo_info tmp;
    rc = walk(data, len, &tmp, NULL, -1, q);
    if (rc) return rc;
    for (c = 0; c < info->ncomp; c++) defined[c] = info->quant_defined[info->tq[c]];
    for (c = 0; c < info->ncomp; c++) {
        memcpy(info->quant[c], q[c], sizeof(q[c]));
        info->quant_defined[c] = defined[c];
        info->tq[c] = c;
    }
    return JPGO_OK;
}

/* ------------------------------------------------------------------------------------------------ */
/* Entropy decode of one scan.  MCU order follows codestream/sequentialscan.cpp:381-428; restart
 * handling follows codestream/entropyparser.hpp:147-160 and entropyparser.cpp:117-199, including the
 * resynchronisation after a missing / out-of-order RSTn.                                              */
static int decode_scan(const uint8_t *d, size_t len, const jpgo_info *info, const jpgo_scan *sc, decoder_tables *tabs,
                       int lowbit, int32_t *const planes[]) {
    bitreader br;
    int32_t pred[JPGO_MAX_COMP] = {0, 0, 0, 0};
    unsigned skip[JPGO_MAX_COMP] = {0, 0, 0, 0};
    int32_t dummy[64];
    const uint8_t *end = d + sc->ecs_end, *file_end = d + len;
    const int progressive = (info->frame_type == 2);
    int valid = 1;
    int total = sc->mcu_cols * sc->mcu_rows;
    int togo = sc->restart_interval, next_rst = 0xd0;
    int m, c;
    for (c = 0; c < sc->ns; c++) { /* a progressive scan only needs the tables it decodes with */
        const int need_dc = !progressive || (sc->ss == 0 && sc->ah == 0), need_ac = !progressive || sc->se != 0;
        if ((need_dc && !tabs->dc[sc->td[c]].defined) || (need_ac && !tabs->ac[sc->ta[c]].defined)) return JPGO_ERR_MALFORMED_STREAM;
    }
    br_open(&br, d + sc->ecs_offset, end);
    for (m = 0; m < total; m++) {
        int mx = m % sc->mcu_cols, my = m / sc->mcu_cols;
        if (sc->restart_interval) {
            if (togo == 0) { /* BeginReadMCU -> ParseRestartMarker, entropyparser.cpp:117-199 */
                const uint8_t *p = br.p;
                while (p + 1 < end && p[0] == 0xff && p[1] == 0xff) p++; /* fill bytes, :121-125 */
                if (p + 1 < end && p[0] == 0xff && p[1] == next_rst) {
                    p += 2;
                    valid = 1;
                } else { /* out of sync: advance to the next marker and decide from its id, :137-199 */
                    valid = -1;
                    while (valid < 0) {
                        while (p < file_end && p[0] != 0xff) p++;
                        if (p + 1 >= file_end) return JPGO_ERR_UNEXPECTED_EOF; /* ran out of data while resynchronising */
                        if (p[1] >= 0xd0 && p[1] <= 0xd7) {
                            if (p[1] == next_rst) { /* the decoder was behind: back in step */
                                p += 2;
                                valid = 1;
                            } else if (((p[1] - next_rst) & 7) >= 4) {
                                p += 2; /* a marker the decoder is already past: drop it, keep looking */
                            } else {
                                valid = 0; /* the marker is ahead: this interval is lost, the marker stays */
                            }
                        } else if (p[1] >= 0xc0 && p[1] < 0xf0) {
                            valid = 0; /* some other marker: the segment is over, everything that follows is lost */
                        } else {
                            p++; /* FF 00 or garbage: eat the FF and go on */
                        }
                    }
                }
                br_open(&br, p, end); /* SequentialScan::Restart, sequentialscan.cpp:266-274 (only read when valid) */
                memset(pred, 0, sizeof(pred));
                memset(skip, 0, sizeof(skip));
                next_rst = 0xd0 + ((next_rst + 1) & 7);
                togo = sc->restart_interval;
            }
            togo--;
        }
        if (!valid) continue; /* the MCUs of an invalid segment are cleared (sequentialscan.cpp:415-419): they stay zero */
        for (c = 0; c < sc->ns; c++) {
            int ci = sc->comp[c];
            int mw = (sc->ns > 1) ? info->hs[ci] : 1, mh = (sc->ns > 1) ? info->vs[ci] : 1;
            int x, y;
            for (y = 0; y < mh; y++) {
                for (x = 0; x < mw; x++) {
                    int bx = mx * mw + x, by = my * mh + y;
                    int32_t *blk = dummy;
                    /* blocks outside the reference's stored grid are decoded and dropped (:407-412);
                     * this oracle keeps the MCU-padded grid, the extra blocks are simply never read back */
                    if (bx < info->bw[ci] && by < info->bh[ci]) blk = planes[ci] + 64 * ((size_t)by * info->bw[ci] + bx);
                    else if (progressive) memset(dummy, 0, sizeof(dummy));
                    if (!progressive) decode_block(blk, &tabs->dc[sc->td[c]], &tabs->ac[sc->ta[c]], &pred[c], lowbit, &br);
                    else if (sc->ah == 0) decode_block_first(blk, &tabs->dc[sc->td[c]], &tabs->ac[sc->ta[c]], &pred[c], sc, &skip[c], &br);
                    else decode_block_refine(blk, &tabs->ac[sc->ta[c]], sc, &skip[c], &br);
                    if (br.error) return br.error;
                }
            }
        }
    }
    return JPGO_OK;
}

static int build_tables(decoder_tables *t) {
    int i, rc;
    for (i = 0; i < 8; i++) {
        hufftab *h = (i < 4) ? &t->dc[i] : &t->ac[i - 4];
        if (!h->defined) continue;
        if (!h->sym2) {
            h->sym2 = (uint8_t *)malloc(65536);
            h->len2 = (uint8_t *)malloc(65536);
            if (!h->sym2 || !h->len2) return JPGO_ERR_OUT_OF_MEMORY;
        }
        rc = jpgo_build_huffman(h->bits, h->vals, h->nvals, h->sym1, h->len1, h->sym2, h->len2, h->has2);
        if (rc) return rc;
    }
    return JPGO_OK;
}

static void free_tables(decoder_tables *t) {
    int i;
    for (i = 0; i < 4; i++) {
        free(t->dc[i].sym2);
        free(t->dc[i].len2);
        free(t->ac[i].sym2);
        free(t->ac[i].len2);
    }
}

int jpgo_decode_coefficients(const uint8_t *data, size_t len, const jpgo_info *info, int32_t *const planes[]) {
    int s, c, rc = JPGO_OK;
    decoder_tables *tabs = (decoder_tables *)calloc(1, sizeof(*tabs));
    jpgo_info tmp;
    if (!tabs) return JPGO_ERR_OUT_OF_MEMORY;
    for (c = 0; c < info->ncomp; c++) memset(planes[c], 0, sizeof(int32_t) * 64 * (size_t)info->bw[c] * info->bh[c]);
    for (s = 0; s < info->nscans && rc == JPGO_OK; s++) {
        /* tables may be redefined between scans: re-walk up to scan s and take what is in effect there */
        free_tables(tabs);
        memset(tabs, 0, sizeof(*tabs));
        rc = walk(data, len, &tmp, tabs, s, NULL);
        if (rc) break;
        rc = build_tables(tabs);
        if (rc) break;
        rc = decode_scan(data, len, info, &info->scan[s], tabs, tabs->lowbit[s], planes);
    }
    free_tables(tabs);
    free(tabs);
    return rc;
}

/* ------------------------------------------------------------------------------------------------ */
/* Dequantisation + inverse DCT.  Follows dct/idct.cpp:98-108 (multiplier = delta << 4) and
 * dct/idct.cpp:226-339 with FIX_BITS = 9, INTERMEDIATE_BITS = 0 (dct/idct.hpp:70-77): pass 1 over the
 * rows rounds with (x + 256) >> 9, pass 2 over the columns with (x + 2048) >> 12; the level shift
 * dcoffset << 7 joins the dequantised DC before pass 1.  Constants are WORD(x * 512 + 0.5).
 * All arithmetic is 32-bit two's complement (unsigned casts make the wrap-around defined in C).      */
#define MUL(a, k) ((int32_t)((uint32_t)(a) * (uint32_t)(int32_t)(k)))
#define ADD(a, b) ((int32_t)((uint32_t)(a) + (uint32_t)(b)))
#define SUB(a, b) ((int32_t)((uint32_t)(a) - (uint32_t)(b)))
#define SHL9(a) ((int32_t)((uint32_t)(a) << 9))

static void idct_1d(const int32_t in[8], int32_t out[8], int32_t round, int shift) {
    int32_t tz2 = in[2], tz3 = in[6];
    int32_t z1 = MUL(ADD(tz2, tz3), 277);
    int32_t tmp2 = ADD(z1, MUL(tz3, -946));
    int32_t tmp3 = ADD(z1, MUL(tz2, 392));
    int32_t tmp0 = SHL9(ADD(in[0], in[4]));
    int32_t tmp1 = SHL9(SUB(in[0], in[4]));
    int32_t tmp10 = ADD(tmp0, tmp3), tmp13 = SUB(tmp0, tmp3);
    int32_t tmp11 = ADD(tmp1, tmp2), tmp12 = SUB(tmp1, tmp2);
    int32_t t0 = in[7], t1 = in[5], t2 = in[3], t3 = in[1];
    int32_t z1o = ADD(t0, t3), z2 = ADD(t1, t2), z3 = ADD(t0, t2), z4 = ADD(t1, t3);
    int32_t z5 = MUL(ADD(z3, z4), 602);
    t0 = MUL(t0, 153);
    t1 = MUL(t1, 1051);
    t2 = MUL(t2, 1573);
    t3 = MUL(t3, 769);
    z1o = MUL(z1o, -461);
    z2 = MUL(z2, -1312);
    z3 = ADD(MUL(z3, -1004), z5);
    z4 = ADD(MUL(z4, -200), z5);
    t0 = ADD(t0, ADD(z1o, z3));
    t1 = ADD(t1, ADD(z2, z4));
    t2 = ADD(t2, ADD(z2, z3));
    t3 = ADD(t3, ADD(z1o, z4));
    out[0] = ADD(ADD(tmp10, t3), round) >> shift;
    out[7] = ADD(SUB(tmp10, t3), round) >> shift;
    out[1] = ADD(ADD(tmp11, t2), round) >> shift;
    out[6] = ADD(SUB(tmp11, t2), round) >> shift;
    out[2] = ADD(ADD(tmp12, t1), round) >> shift;
    out[5] = ADD(SUB(tmp12, t1), round) >> shift;
    out[3] = ADD(ADD(tmp13, t0), round) >> shift;
    out[4] = ADD(SUB(tmp13, t0), round) >> shift;
}

void jpgo_idct_block(int32_t *target, const int32_t *source, const uint16_t *delta, int32_t dcoffset) {
    int32_t tmp[64];
    int r, c, i;
    if (!source) { /* idct.cpp:336-338 */
        memset(target, 0, 64 * sizeof(int32_t));
        return;
    }
    for (r = 0; r < 8; r++) {
        int32_t in[8];
        for (i = 0; i < 8; i++) in[i] = MUL(source[8 * r + i], (int32_t)delta[8 * r + i] << 4);
        if (r == 0) in[0] = ADD(in[0], (int32_t)((uint32_t)dcoffset << 7)); /* :233,244 */
        idct_1d(in, tmp + 8 * r, 256, 9);
    }
    for (c = 0; c < 8; c++) {
        int32_t in[8], out[8];
        for (i = 0; i < 8; i++) in[i] = tmp[8 * i + c];
        idct_1d(in, out, 2048, 12);
        for (i = 0; i < 8; i++) target[8 * i + c] = out[i];
    }
}

/* ------------------------------------------------------------------------------------------------ */
/* Reconstruction: control/blockbitmaprequester.cpp:1249-1272 (ReconstructRegion), :1079-1112
 * (PullQData), :1151-1224 (PushReconstructedData), :1013-1074 (ReconstructUnsampled).
 * Sample planes are int32 carrying 4 fractional bits ("COLOR_BITS", colortrafo/colortrafo.hpp:70-73). */

/* The component's IDCT output as the upsampler line buffer sees it: upsampling/upsamplerbase.cpp:61-76
 * (width = ceil(W/sx), lines = ceil(H/sy)), :300-327 (every line gets dest[-1] = dest[0] and
 * dest[width] = dest[width-1]).  Stored here as plane[(y)*(pw) + 1 + x] with pw = 8*bw + 2.           */
typedef struct {
    int32_t *s;
    int pw;     /* pitch */
    int w, h;   /* true subsampled size */
} splane;

static int32_t sp_at(const splane *p, int x, int y) { /* x in [-1, w] after edge replication */
    return p->s[(size_t)y * p->pw + 1 + x];
}

/* Upsampler<sx,sy>::UpsampleRegion for one 8x8 output block whose top-left output pixel is (X,Y):
 * upsampling/upsampler.cpp:83-112, VerticalFilterCore<1..4> :114-268, HorizontalFilterCore<1..4> :270-386.
 * The weights are (1,3)/4 for factors 2 and 3 (3: every third line / column is the sample itself) and
 * (3,5)/8, (1,7)/8 for factor 4; the rounding constant alternates between neighbouring columns / lines.
 * The horizontal cores work IN PLACE on the row (input shifted by one pixel), so a few outputs read
 * positions that were already overwritten -- that is part of the contract and is reproduced by doing
 * the same stores in the same order.  out[8*row + col].                                              */
static int32_t mix(int32_t a, int wa, int32_t b, int wb, int rnd, int sh) { return ADD(ADD(MUL(wa, a), MUL(wb, b)), rnd) >> sh; }

static void upsample_block(const splane *p, int sx, int sy, int X, int Y, int32_t *out) {
    int y = Y / sy;
    int x0 = X / sx - ((sx > 1) ? 1 : 0); /* window col 0; one extra pixel on the left when expanding */
    int row, j;
    int top = (y > 0) ? y - 1 : y, cur = y, bot = (y + 1 < p->h) ? y + 1 : y;
    int ymod = Y % sy, xmod = X % sx;
    for (row = 0; row < 8; row++) {
        int32_t *o = out + 8 * row;
        int advance = 0;
        /* ---- vertical: line `cur` leaning on `top` in the upper part of its sy output lines, on `bot` in the lower */
        if (sy == 1) {
            for (j = 0; j < 8; j++) o[j] = sp_at(p, x0 + j, cur);
            if (cur + 1 < p->h) cur++;
        } else if (sy == 2) {
            const int nb = (ymod == 0) ? top : bot;
            for (j = 0; j < 8; j++) o[j] = mix(sp_at(p, x0 + j, nb), 1, sp_at(p, x0 + j, cur), 3, ((j & 1) == ymod) ? 2 : 1, 2);
            advance = (ymod == 1);
        } else if (sy == 3) {
            if (ymod == 1) {
                for (j = 0; j < 8; j++) o[j] = sp_at(p, x0 + j, cur);
            } else {
                const int nb = (ymod == 0) ? top : bot;
                for (j = 0; j < 8; j++) o[j] = mix(sp_at(p, x0 + j, nb), 1, sp_at(p, x0 + j, cur), 3, (((j & 1) == 0) == (ymod == 0)) ? 2 : 1, 2);
            }
            advance = (ymod == 2);
        } else { /* sy == 4 */
            const int nb = (ymod < 2) ? top : bot, far = (ymod == 0 || ymod == 3); /* far from the sample line: 3:5, else 1:7 */
            for (j = 0; j < 8; j++) {
                int rnd;
                if (ymod == 0 || ymod == 2 || ymod == 3) rnd = (j & 1) ? 3 : 4;
                else rnd = (j & 1) ? 4 : 3;
                o[j] = mix(sp_at(p, x0 + j, nb), far ? 3 : 1, sp_at(p, x0 + j, cur), far ? 5 : 7, rnd, 3);
            }
            advance = (ymod == 3);
        }
        if (sy > 1) {
            if (advance) {
                ymod = 0;
                top = cur;
                cur = bot;
                if (bot + 1 < p->h) bot++;
            } else {
                ymod++;
            }
        }
        /* ---- horizontal, in place, in the reference's store order */
        if (sx == 2) {
            int32_t *src = o + 1, t;
            o[7] = mix(src[4], 1, src[3], 3, 1, 2);
            o[6] = mix(src[2], 1, src[3], 3, 2, 2);
            o[5] = mix(src[3], 1, src[2], 3, 1, 2);
            o[4] = mix(src[1], 1, src[2], 3, 2, 2);
            o[3] = mix(src[2], 1, src[1], 3, 1, 2);
            o[2] = mix(src[0], 1, src[1], 3, 2, 2);
            t = src[0];
            o[1] = mix(src[1], 1, t, 3, 1, 2); /* src[1] is the NEW o[2] */
            o[0] = mix(src[-1], 1, t, 3, 2, 2);
        } else if (sx == 3) {
            int32_t *src = o + 1, t;
            if (xmod == 0) {
                o[7] = src[2];
                o[6] = mix(src[1], 1, src[2], 3, 2, 2);
                o[5] = mix(src[2], 1, src[1], 3, 1, 2);
                o[4] = src[1];
                o[3] = mix(src[0], 1, src[1], 3, 2, 2);
                o[2] = mix(src[1], 1, src[0], 3, 1, 2);
                o[0] = mix(src[-1], 1, src[0], 3, 2, 2);
                o[1] = src[0];
            } else if (xmod == 1) {
                o[7] = mix(src[3], 1, src[2], 3, 1, 2);
                o[6] = src[2];
                o[5] = mix(src[1], 1, src[2], 3, 2, 2);
                o[4] = mix(src[2], 1, src[1], 3, 1, 2);
                o[3] = src[1];
                t = src[0];
                o[2] = mix(t, 1, src[1], 3, 2, 2);
                o[1] = mix(src[1], 1, t, 3, 1, 2);
                o[0] = t;
            } else {
                o[7] = mix(src[2], 1, src[3], 3, 2, 2);
                o[6] = mix(src[3], 1, src[2], 3, 1, 2);
                o[5] = src[2];
                o[4] = mix(src[1], 1, src[2], 3, 2, 2);
                o[3] = mix(src[2], 1, src[1], 3, 1, 2);
                o[2] = src[1];
                t = src[0];
                o[1] = mix(t, 1, src[1], 3, 2, 2);
                o[0] = mix(src[1], 1, t, 3, 1, 2);
            }
        } else if (sx == 4) {
            int32_t *src = o + 1, t;
            o[7] = mix(src[2], 3, src[1], 5, 1, 3);
            o[6] = mix(src[2], 1, src[1], 7, 2, 3);
            o[5] = mix(src[0], 1, src[1], 7, 1, 3);
            o[4] = mix(src[0], 3, src[1], 5, 2, 3);
            t = src[0];
            o[3] = mix(src[1], 3, t, 5, 1, 3);
            o[2] = mix(src[1], 1, t, 7, 2, 3);
            o[1] = mix(src[-1], 1, t, 7, 1, 3);
            o[0] = mix(src[-1], 3, t, 5, 2, 3);
        }
    }
}

static int64_t clampmax(int64_t v, int64_t max) { return v < 0 ? 0 : (v > max ? max : v); } /* CLAMP(max, v), ycbcrtrafo.cpp:61 */

/* out8 for 8-bit frames (one byte per sample) or out16 (native-endian 16-bit samples, any precision): what the
 * reference writes for CTYP_UBYTE / CTYP_UWORD client bitmaps. Level shift, chroma offset and clamp scale with the
 * precision (1 << (precision - 1), (1 << precision) - 1); the arithmetic is the same (tables.cpp:1877-1891: the LONG
 * IDCT up to 12 bits).                                                                                  */
/* IDCT of every stored block into a sample plane (what PullQData/DefineRegion or the direct IDCT produce), with the edge
 * columns the upsampler replicates (upsamplerbase.cpp:322-323) */
static int build_sample_planes(const jpgo_info *info, int32_t *const planes[], splane sp[JPGO_MAX_COMP]) {
    const int32_t dcshift = (int32_t)1 << (info->precision - 1);
    int c, bx, by, i;
    int W = info->width, H = info->height, nc = info->ncomp;
    memset(sp, 0, sizeof(splane) * JPGO_MAX_COMP);
    for (c = 0; c < nc; c++)
        if (!info->quant_defined[info->tq[c]]) return JPGO_ERR_MALFORMED_STREAM;
    for (c = 0; c < nc; c++) {
        splane *p = &sp[c];
        p->w = (W + info->subx[c] - 1) / info->subx[c];
        p->h = (H + info->suby[c] - 1) / info->suby[c];
        p->pw = 8 * info->bw[c] + 2 + 8;
        p->s = (int32_t *)calloc((size_t)p->pw * 8 * info->bh[c], sizeof(int32_t));
        if (!p->s) return JPGO_ERR_OUT_OF_MEMORY;
        for (by = 0; by < info->bh[c]; by++) {
            for (bx = 0; bx < info->bw[c]; bx++) {
                int32_t blk[64];
                int r;
                /* blocks outside the reference's stored grid do not exist there; they only ever feed
                 * samples at x >= w or y >= h, which the edge replication below overwrites / nobody reads */
                jpgo_idct_block(blk, planes[c] + 64 * ((size_t)by * info->bw[c] + bx), info->quant[info->tq[c]], dcshift);
                for (r = 0; r < 8; r++) memcpy(p->s + (size_t)(8 * by + r) * p->pw + 1 + 8 * bx, blk + 8 * r, 32);
            }
        }
        for (i = 0; i < 8 * info->bh[c]; i++) { /* upsamplerbase.cpp:322-323 */
            int32_t *line = p->s + (size_t)i * p->pw + 1;
            line[-1] = line[0];
            line[p->w] = line[p->w - 1];
        }
    }
    return JPGO_OK;
}

/* the 8x8 output block (bx, by) of every component, upsampled to the frame's resolution, 4 fractional bits */
static void block_samples(const jpgo_info *info, const splane sp[JPGO_MAX_COMP], int bx, int by, int32_t buf[JPGO_MAX_COMP][64]) {
    int c, x, y;
    for (c = 0; c < info->ncomp; c++) {
        if (info->subx[c] > 1 || info->suby[c] > 1) {
            upsample_block(&sp[c], info->subx[c], info->suby[c], 8 * bx, 8 * by, buf[c]);
        } else {
            for (y = 0; y < 8; y++)
                for (x = 0; x < 8; x++) buf[c][8 * y + x] = sp[c].s[(size_t)(8 * by + y) * sp[c].pw + 1 + 8 * bx + x];
        }
    }
}

static int reconstruct(const jpgo_info *info, int32_t *const planes[], uint8_t *out8, uint16_t *out16) {
    const int32_t dcshift = (int32_t)1 << (info->precision - 1);
    const int64_t maxval = ((int64_t)1 << info->precision) - 1;
    splane sp[JPGO_MAX_COMP];
    int c, rc, bx, by;
    int W = info->width, H = info->height, nc = info->ncomp;
    rc = build_sample_planes(info, planes, sp);
    if (rc) goto done;
    for (by = 0; by < (H + 7) / 8; by++) {
        for (bx = 0; bx < (W + 7) / 8; bx++) {
            int32_t buf[JPGO_MAX_COMP][64];
            int xmax = (8 * bx + 7 < W) ? 7 : (W - 1) & 7, ymax = (8 * by + 7 < H) ? 7 : (H - 1) & 7, x, y;
            block_samples(info, sp, bx, by, buf);
            /* YCbCrTrafo<UBYTE,count,ClampFlag,trafo,Zero>::YCbCr2RGB, colortrafo/ycbcrtrafo.cpp:679-1008 */
            for (y = 0; y <= ymax; y++) {
                for (x = 0; x <= xmax; x++) {
                    const size_t at = ((size_t)(8 * by + y) * W + (8 * bx + x)) * nc;
                    int64_t v[JPGO_MAX_COMP];
                    if (nc == 3 && info->ycbcr) { /* :842-850, matrix colortransformerfactory.cpp:136-138 */
                        int64_t yv = buf[0][8 * y + x];
                        int64_t cb = (int64_t)buf[1][8 * y + x] - ((int64_t)dcshift << 4);
                        int64_t cr = (int64_t)buf[2][8 * y + x] - ((int64_t)dcshift << 4);
                        v[0] = clampmax((yv * 8192 + cb * 0 + cr * 11485 + 65536) >> 17, maxval);
                        v[1] = clampmax((yv * 8192 + cb * -2819 + cr * -5850 + 65536) >> 17, maxval);
                        v[2] = clampmax((yv * 8192 + cb * 14516 + cr * 0 + 65536) >> 17, maxval);
                    } else { /* identity: COLOR_TO_INT, tools/numerics.hpp:69 */
                        for (c = 0; c < nc; c++) v[c] = clampmax(((int64_t)buf[c][8 * y + x] + 8) >> 4, maxval);
                    }
                    for (c = 0; c < nc; c++) {
                        if (out16) out16[at + c] = (uint16_t)v[c];
                        else out8[at + c] = (uint8_t)v[c];
                    }
                }
            }
        }
    }
done:
    for (c = 0; c < nc; c++) free(sp[c].s);
    return rc;
}

int jpgo_reconstruct(const jpgo_info *info, int32_t *const planes[], uint8_t *out) {
    if (info->precision != 8) return JPGO_ERR_INVALID_PARAMETER; /* one byte per sample only holds 8-bit frames */
    return reconstruct(info, planes, out, NULL);
}

int jpgo_reconstruct16(const jpgo_info *info, int32_t *const planes[], uint16_t *out) { return reconstruct(info, planes, NULL, out); }

/* JPGTAG_DECODER_UPSAMPLE = false (control/bitmapctrl.cpp:273-293, BlockBitmapRequester::ReconstructUnsampled,
 * control/blockbitmaprequester.cpp:1013-1074): one component per request at its own resolution, no upsampling, the identity
 * "colour transformation" (the reference refuses anything else).  Component c is written as a plane of
 * ceil(W/subx) x ceil(H/suby) native-endian 16-bit samples at out + (sum of the planes before it). */
int jpgo_reconstruct_planes16(const jpgo_info *info, int32_t *const planes[], uint16_t *out) {
    const int32_t dcshift = (int32_t)1 << (info->precision - 1);
    const int64_t maxval = ((int64_t)1 << info->precision) - 1;
    int c, bx, by, x, y;
    for (c = 0; c < info->ncomp; c++) {
        const int w = (info->width + info->subx[c] - 1) / info->subx[c], h = (info->height + info->suby[c] - 1) / info->suby[c];
        if (!info->quant_defined[info->tq[c]]) return JPGO_ERR_MALFORMED_STREAM;
        for (by = 0; by < (h + 7) / 8; by++)
            for (bx = 0; bx < (w + 7) / 8; bx++) {
                int32_t blk[64];
                jpgo_idct_block(blk, planes[c] + 64 * ((size_t)by * info->bw[c] + bx), info->quant[info->tq[c]], dcshift);
                for (y = 0; y < 8 && 8 * by + y < h; y++)
                    for (x = 0; x < 8 && 8 * bx + x < w; x++) /* COLOR_TO_INT, tools/numerics.hpp:69 */
                        out[(size_t)(8 * by + y) * w + 8 * bx + x] = (uint16_t)clampmax(((int64_t)blk[8 * y + x] + 8) >> 4, maxval);
            }
        out += (size_t)w * h;
    }
    return JPGO_OK;
}

int jpgo_decode_planes16(const uint8_t *data, size_t len, uint16_t *out, size_t cap_samples, jpgo_info *info_out) {
    jpgo_info info;
    int32_t *planes[JPGO_MAX_COMP] = {0, 0, 0, 0};
    size_t need = 0;
    int rc, c;
    rc = jpgo_read_info(data, len, &info);
    if (info_out) *info_out = info;
    if (rc) return rc;
    for (c = 0; c < info.ncomp; c++)
        need += (size_t)((info.width + info.subx[c] - 1) / info.subx[c]) * ((info.height + info.suby[c] - 1) / info.suby[c]);
    if (cap_samples < need) return JPGO_ERR_INVALID_PARAMETER;
    for (c = 0; c < info.ncomp; c++) {
        planes[c] = (int32_t *)malloc(sizeof(int32_t) * 64 * (size_t)info.bw[c] * info.bh[c]);
        if (!planes[c]) rc = JPGO_ERR_OUT_OF_MEMORY;
    }
    if (!rc) rc = jpgo_decode_coefficients(data, len, &info, planes);
    if (!rc) rc = latched_quantisers(data, len, &info);
    if (!rc) rc = jpgo_reconstruct_planes16(&info, planes, out);
    for (c = 0; c < info.ncomp; c++) free(planes[c]);
    return rc;
}

static int decode_any(const uint8_t *data, size_t len, uint8_t *out8, uint16_t *out16, size_t cap, jpgo_info *info_out);

int jpgo_decode(const uint8_t *data, size_t len, uint8_t *out, size_t cap, jpgo_info *info_out) {
    return decode_any(data, len, out, NULL, cap, info_out);
}

int jpgo_decode16(const uint8_t *data, size_t len, uint16_t *out, size_t cap_samples, jpgo_info *info_out) {
    return decode_any(data, len, NULL, out, cap_samples, info_out);
}

/* ------------------------------------------------------------------------------------------------ */
/* JPEG XT (ISO/IEC 18477) residual layer, SURVEY 8f3 -- the integer profile the reference encoder writes with
 * `-r -q <base> -Q <extension>` for 8-bit images: a second, ordinary DCT codestream in a RESI box of the APP11 markers,
 * merged pixel by pixel with the base image (YCbCrTrafo::YCbCr2RGB, colortrafo/ycbcrtrafo.cpp:747-880) under the control of
 * the merging specification box SPEC.  Boxes: boxes/box.cpp:95-205 (APP11: 'JP', enumerator, sequence number, LBox, TBox,
 * payload; pieces of one box are concatenated), boxes/superbox.cpp (SPEC holds sub-boxes LBox TBox payload),
 * boxes/outputconversionbox.cpp:92-127, boxes/colortrafobox.cpp:55-78.  Everything outside that profile -- tone mapping
 * curves, free-form matrices, refinement scans, the lossless / DCT-bypass residuals, alpha, float output -- is reported as
 * NOT_IMPLEMENTED, never decoded as if it were absent.                                                             */
typedef struct {
    int have_spec, have_resi, unsupported;
    uint8_t *spec, *resi;
    size_t spec_len, resi_len, spec_size, resi_size; /* collected so far / LBox - 8 */
    int spec_en, resi_en;
    int ocon, ltrf, rtrf, ctrf; /* first byte of the sub-box payload, -1 = absent */
} xt_boxes;

static void xt_free(xt_boxes *x) {
    free(x->spec);
    free(x->resi);
    x->spec = x->resi = NULL;
}

static uint32_t rd32(const uint8_t *p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
#define XT_ID(a, b, c, d) (((uint32_t)(a) << 24) | ((uint32_t)(b) << 16) | ((uint32_t)(c) << 8) | (uint32_t)(d))

/* collects the SPEC and RESI boxes of the APP11 markers in front of the first scan */
static int xt_collect(const uint8_t *d, size_t n, xt_boxes *x) {
    size_t pos = 2;
    memset(x, 0, sizeof(*x));
    x->ocon = x->ltrf = x->rtrf = x->ctrf = -1;
    if (n < 4 || d[0] != 0xff || d[1] != 0xd8) return JPGO_OK;
    while (pos + 3 < n && d[pos] == 0xff) {
        int m = d[pos + 1];
        size_t len;
        if (m == 0xff) {
            pos++;
            continue;
        }
        if (m == 0xda || m == 0xd9) break;
        if (m >= 0xd0 && m <= 0xd7) {
            pos += 2;
            continue;
        }
        len = ((size_t)d[pos + 2] << 8) | d[pos + 3];
        if (len < 2 || pos + 2 + len > n) break;
        if (m == 0xeb && len >= 2 + 2 + 2 + 4 + 4 + 4 && d[pos + 4] == 'J' && d[pos + 5] == 'P') {
            const uint8_t *b = d + pos + 6;
            const int en = (b[0] << 8) | b[1];
            const uint32_t lbox = rd32(b + 6), tbox = rd32(b + 10);
            const uint8_t *payload = b + 14;
            const size_t plen = len - 2 - 2 - 2 - 4 - 4 - 4;
            uint8_t **buf = NULL;
            size_t *have = NULL, *size = NULL;
            int *ben = NULL, *flag = NULL;
            if (tbox == XT_ID('S', 'P', 'E', 'C')) buf = &x->spec, have = &x->spec_len, size = &x->spec_size, ben = &x->spec_en, flag = &x->have_spec;
            else if (tbox == XT_ID('R', 'E', 'S', 'I')) buf = &x->resi, have = &x->resi_len, size = &x->resi_size, ben = &x->resi_en, flag = &x->have_resi;
            else if (tbox != XT_ID('f', 't', 'y', 'p') && tbox != XT_ID('L', 'C', 'H', 'K')) x->unsupported = 1; /* refinement, alpha, curves, matrices ... */
            if (buf) {
                if (lbox < 8) { /* 1 = XLBox (boxes beyond 4 GB), 0 = to the end of the file */
                    x->unsupported = 1;
                } else if (!*flag) {
                    *flag = 1;
                    *ben = en;
                    *size = lbox - 8;
                    *buf = (uint8_t *)malloc(*size ? *size : 1);
                    if (!*buf) return JPGO_ERR_OUT_OF_MEMORY;
                } else if (*ben != en || *size != lbox - 8) {
                    x->unsupported = 1; /* a second box of this type */
                    buf = NULL;
                }
                if (buf && *buf) {
                    if (*have + plen > *size) return JPGO_ERR_MALFORMED_STREAM; /* box.cpp:186-188 */
                    memcpy(*buf + *have, payload, plen);
                    *have += plen;
                }
            }
        }
        pos += 2 + len;
    }
    if ((x->have_spec && x->spec_len != x->spec_size) || (x->have_resi && x->resi_len != x->resi_size)) return JPGO_ERR_MALFORMED_STREAM;
    if (x->have_spec) { /* the sub-boxes of the merging specification */
        size_t p = 0;
        while (p + 8 <= x->spec_len) {
            const uint32_t lbox = rd32(x->spec + p), tbox = rd32(x->spec + p + 4);
            if (lbox < 8 || p + lbox > x->spec_len) return JPGO_ERR_MALFORMED_STREAM;
            if (tbox == XT_ID('O', 'C', 'O', 'N') && lbox == 11) x->ocon = x->spec[p + 8] | (x->spec[p + 9] << 8) | (x->spec[p + 10] << 16);
            else if (tbox == XT_ID('L', 'T', 'R', 'F') && lbox == 9) x->ltrf = x->spec[p + 8];
            else if (tbox == XT_ID('R', 'T', 'R', 'F') && lbox == 9) x->rtrf = x->spec[p + 8];
            else if (tbox == XT_ID('C', 'T', 'R', 'F') && lbox == 9) x->ctrf = x->spec[p + 8];
            else x->unsupported = 1;
            p += lbox;
        }
        if (p != x->spec_len) return JPGO_ERR_MALFORMED_STREAM;
    }
    return JPGO_OK;
}

/* Base image + residual image -> pixels.  Parameters of the 8-bit integer profile (colortransformerfactory.cpp:686-705,
 * 300-352, 425-520): max = rmax = outmax = 255, DC shifts 128; L tables the identity over 0..255 (a lookup clamps its index),
 * the C transformation the identity, Q tables the identity over the pre-shifted range 0..4095, R2 tables
 * floor(i / 16 + 0.5) over 0..4095 (ParametricToneMappingBox::ScaledTableOf, boxes/parametrictonemappingbox.cpp:387-426),
 * clamping output (OCON flag 0x02).                                                                              */
static int xt_merge(const jpgo_info *bi, int32_t *const bplanes[], const jpgo_info *ri, int32_t *const rplanes[], int l_ycbcr, int r_ycbcr,
                    uint8_t *out8, uint16_t *out16) {
    splane bs[JPGO_MAX_COMP], rs[JPGO_MAX_COMP];
    int c, rc, bx, by;
    const int W = bi->width, H = bi->height, nc = bi->ncomp;
    memset(rs, 0, sizeof(rs));
    rc = build_sample_planes(bi, bplanes, bs);
    if (!rc) rc = build_sample_planes(ri, rplanes, rs);
    if (rc) goto done;
    for (by = 0; by < (H + 7) / 8; by++) {
        for (bx = 0; bx < (W + 7) / 8; bx++) {
            int32_t b[JPGO_MAX_COMP][64], r[JPGO_MAX_COMP][64];
            int xmax = (8 * bx + 7 < W) ? 7 : (W - 1) & 7, ymax = (8 * by + 7 < H) ? 7 : (H - 1) & 7, x, y;
            block_samples(bi, bs, bx, by, b);
            block_samples(ri, rs, bx, by, r);
            for (y = 0; y <= ymax; y++) {
                for (x = 0; x <= xmax; x++) {
                    const size_t at = ((size_t)(8 * by + y) * W + (8 * bx + x)) * nc;
                    const int i = 8 * y + x;
                    int64_t res[3] = {128, 128, 128}, v[3] = {0, 0, 0};
                    /* the residual: Q table first (clamped index), then the R transformation, then the R2 table
                     * (ycbcrtrafo.cpp:757-828) */
                    if (nc == 3 && r_ycbcr) {
                        const int64_t yv = clampmax(r[0][i], 4095), cb = clampmax(r[1][i], 4095) - (128 << 4), cr = clampmax(r[2][i], 4095) - (128 << 4);
                        res[0] = (yv * 8192 + cr * 11485 + 4096) >> 13; /* FIX_COLOR_TO_INTCOLOR, tools/numerics.hpp:67 */
                        res[1] = (yv * 8192 - cb * 2819 - cr * 5850 + 4096) >> 13;
                        res[2] = (yv * 8192 + cb * 14516 + 4096) >> 13;
                    } else {
                        for (c = 0; c < nc; c++) res[c] = clampmax(r[c][i], 4095);
                    }
                    for (c = 0; c < nc; c++) res[c] = (clampmax(res[c], 4095) + 8) >> 4;
                    /* the base image: L transformation, then the L table (:834-862) */
                    if (nc == 3 && l_ycbcr) {
                        const int64_t yv = b[0][i], cb = (int64_t)b[1][i] - (128 << 4), cr = (int64_t)b[2][i] - (128 << 4);
                        v[0] = (yv * 8192 + cr * 11485 + 65536) >> 17;
                        v[1] = (yv * 8192 - cb * 2819 - cr * 5850 + 65536) >> 17;
                        v[2] = (yv * 8192 + cb * 14516 + 65536) >> 17;
                    } else {
                        for (c = 0; c < nc; c++) v[c] = ((int64_t)b[c][i] + 8) >> 4;
                    }
                    for (c = 0; c < nc; c++) {
                        /* L table (index clamped), C = identity (FIX_TO_INT(v << 13) = v), merge, clamp (:863-878, :935-947) */
                        const int64_t o = clampmax(clampmax(v[c], 255) + res[c] - 128, 255);
                        if (out16) out16[at + c] = (uint16_t)o;
                        else out8[at + c] = (uint8_t)o;
                    }
                }
            }
        }
    }
done:
    for (c = 0; c < nc; c++) {
        free(bs[c].s);
        free(rs[c].s);
    }
    return rc;
}

static int decode_plain(const uint8_t *data, size_t len, const jpgo_info *info, int32_t *planes[JPGO_MAX_COMP]) {
    int c, rc = JPGO_OK;
    for (c = 0; c < info->ncomp; c++) {
        planes[c] = (int32_t *)malloc(sizeof(int32_t) * 64 * (size_t)info->bw[c] * info->bh[c]);
        if (!planes[c]) rc = JPGO_ERR_OUT_OF_MEMORY;
    }
    if (!rc) rc = jpgo_decode_coefficients(data, len, info, planes);
    return rc;
}

static int decode_xt(const uint8_t *data, size_t len, const jpgo_info *info, const xt_boxes *x, uint8_t *out8, uint16_t *out16) {
    jpgo_info rinfo;
    int32_t *bp[JPGO_MAX_COMP] = {0, 0, 0, 0}, *rp[JPGO_MAX_COMP] = {0, 0, 0, 0};
    int rc, c, l_ycbcr, r_ycbcr;
    const int nc = info->ncomp;
    /* what this restatement covers of MergingSpecBox / ColorTransformerFactory::BuildColorTransformer */
    if (x->unsupported || !x->have_spec || info->precision != 8 || (nc != 1 && nc != 3)) return JPGO_ERR_NOT_IMPLEMENTED;
    if (x->ocon != 0x02) return JPGO_ERR_NOT_IMPLEMENTED;                      /* clamping only: no lossless, float, lookup, extra bits */
    if (x->ctrf != -1 && x->ctrf != (1 << 4)) return JPGO_ERR_NOT_IMPLEMENTED; /* C: identity */
    if (nc == 1) {
        if (x->ltrf != -1) return JPGO_ERR_MALFORMED_STREAM; /* tables.cpp:2001-2003 */
        if (x->rtrf != -1 && x->rtrf != (1 << 4)) return JPGO_ERR_NOT_IMPLEMENTED;
        l_ycbcr = r_ycbcr = 0;
    } else {
        if (x->ltrf == -1) l_ycbcr = info->ycbcr; /* the JPEG default, tables.cpp:2023-2030 */
        else if (x->ltrf == (2 << 4)) l_ycbcr = 1;
        else if (x->ltrf == (1 << 4)) l_ycbcr = 0;
        else return JPGO_ERR_NOT_IMPLEMENTED;
        if (x->rtrf == -1 || x->rtrf == (2 << 4)) r_ycbcr = 1; /* tables.cpp:2052-2060 */
        else if (x->rtrf == (1 << 4)) r_ycbcr = 0;
        else return JPGO_ERR_NOT_IMPLEMENTED; /* RCT (lossless), free form */
    }
    if (!x->have_resi) {
        /* a merging specification without a residual codestream (the reference encoder writes one into every grey file):
         * Extended | ClampFlag, rr = the DC shift: the plain decode with the L transformation the box names (:834-878) */
        jpgo_info plain = *info;
        if (nc == 3) plain.ycbcr = l_ycbcr;
        rc = decode_plain(data, len, &plain, bp);
        if (!rc) rc = reconstruct(&plain, bp, out8, out16);
        for (c = 0; c < nc; c++) free(bp[c]);
        return rc;
    }
    rc = jpgo_read_info(x->resi, x->resi_len, &rinfo); /* residual scan types 0xffb1.. are not ordinary frames: NOT_IMPLEMENTED */
    if (rc) return rc;
    if (rinfo.width != info->width || rinfo.height != info->height || rinfo.ncomp != nc || rinfo.precision != 8) return JPGO_ERR_NOT_IMPLEMENTED;
    rc = decode_plain(data, len, info, bp);
    if (!rc) rc = decode_plain(x->resi, x->resi_len, &rinfo, rp);
    if (!rc) rc = xt_merge(info, bp, &rinfo, rp, l_ycbcr, r_ycbcr, out8, out16);
    for (c = 0; c < nc; c++) {
        free(bp[c]);
        free(rp[c]);
    }
    return rc;
}

/* 1: the stream carries a merging specification (the caller decides what to do about it) */
int jpgo_has_xt_layer(const uint8_t *data, size_t len) {
    xt_boxes x;
    int rc = xt_collect(data, len, &x), yes = (rc != JPGO_OK) || x.have_resi || x.unsupported;
    xt_free(&x);
    return yes;
}

static int decode_any(const uint8_t *data, size_t len, uint8_t *out8, uint16_t *out16, size_t cap, jpgo_info *info_out) {
    jpgo_info info;
    int32_t *planes[JPGO_MAX_COMP] = {0, 0, 0, 0};
    int rc, c;
    rc = jpgo_read_info(data, len, &info);
    if (info_out) *info_out = info;
    if (rc) return rc;
    if (cap < (size_t)info.width * info.height * info.ncomp) return JPGO_ERR_INVALID_PARAMETER;
    {
        xt_boxes x;
        rc = xt_collect(data, len, &x);
        if (!rc && (x.have_spec || x.have_resi || x.unsupported)) {
            rc = (out8 && info.precision != 8) ? JPGO_ERR_INVALID_PARAMETER : decode_xt(data, len, &info, &x, out8, out16);
            xt_free(&x);
            return rc;
        }
        xt_free(&x);
        if (rc) return rc;
    }
    for (c = 0; c < info.ncomp; c++) {
        planes[c] = (int32_t *)malloc(sizeof(int32_t) * 64 * (size_t)info.bw[c] * info.bh[c]);
        if (!planes[c]) rc = JPGO_ERR_OUT_OF_MEMORY;
    }
    if (!rc) rc = jpgo_decode_coefficients(data, len, &info, planes);
    if (!rc) rc = latched_quantisers(data, len, &info);
    if (!rc) rc = out16 ? jpgo_reconstruct16(&info, planes, out16) : jpgo_reconstruct(&info, planes, out8);
    for (c = 0; c < info.ncomp; c++) free(planes[c]);
    return rc;
}
