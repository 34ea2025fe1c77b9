// synth_encoder.cpp -- generator of synthetic baseline-JPEG codestreams (benchmark / test INPUTS only).
//
// The decode path needs restart-partitioned SOF0 streams of the reference-encoder flavour to chew on, on
// machines where neither the reference nor any JPEG library exists (the GPU box).  This is a small,
// self-contained baseline encoder that emits the same stream layout the reference's encoder produces for
// `jpeg -q Q -bl -s 1x1,2x2,2x2 -z DRI` (SURVEY.md 8c): SOI, APP0(JFIF), DQT(two 8-bit tables), DRI, SOF0 with
// component ids 0,1,2, one DHT segment with the four Annex-K tables, SOS, entropy coded data with RSTn markers,
// each interval padded with 1-bits (and a stuffed 00 when the pad byte is FF, io/bitstream.hpp:212-238), EOI.
// Quantisation tables are the Annex-K tables scaled like marker/quantization.cpp:296-299,411.
// It is NOT part of the decode path and is not a port of the reference's encoder (float DCT, box chroma
// downsampling): decode parity is defined on whatever bytes go in.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

namespace {

const uint8_t kZZ[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                         41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                         30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ITU-T T.81 Annex K.1 / K.2 (raster order)
const uint8_t kLumaQ[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                            14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                            18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                            49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
const uint8_t kChromaQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
                              99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                              99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};

// Annex K.3 typical Huffman tables
const uint8_t kDcLumBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
const uint8_t kDcChrBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
const uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
const uint8_t kAcLumBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
const uint8_t kAcLumVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
    0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
    0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
    0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
    0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
    0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
const uint8_t kAcChrBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
const uint8_t kAcChrVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
    0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
    0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
    0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
    0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
    0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
    0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
    0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

struct HuffEnc {
    uint16_t code[256];
    uint8_t len[256];
    void build(const uint8_t *bits, const uint8_t *vals) {
        memset(len, 0, sizeof(len));
        uint32_t c = 0;
        int k = 0;
        for (int l = 1; l <= 16; l++) {
            for (int i = 0; i < bits[l - 1]; i++) {
                code[vals[k]] = (uint16_t)c++;
                len[vals[k]] = (uint8_t)l;
                k++;
            }
            c <<= 1;
        }
    }
};

struct BitWriter {
    std::vector<uint8_t> &out;
    uint64_t acc = 0;
    int n = 0;
    explicit BitWriter(std::vector<uint8_t> &o) : out(o) {}
    void put(uint32_t v, int bits) {
        acc = (acc << bits) | (v & ((1u << bits) - 1u));
        n += bits;
        while (n >= 8) {
            uint8_t b = (uint8_t)(acc >> (n - 8));
            out.push_back(b);
            if (b == 0xff) out.push_back(0);
            n -= 8;
        }
    }
    void flush() {
        if (n > 0) {
            uint8_t b = (uint8_t)((acc << (8 - n)) | ((1u << (8 - n)) - 1u));
            out.push_back(b);
            if (b == 0xff) out.push_back(0);
            n = 0;
        }
        acc = 0;
    }
};

struct DctBasis {
    float c[8][8];
    DctBasis() {
        for (int k = 0; k < 8; k++)
            for (int x = 0; x < 8; x++) c[k][x] = (k == 0 ? std::sqrt(0.125f) : 0.5f) * std::cos((2 * x + 1) * k * 3.14159265358979323846f / 16);
    }
};

void fdct8x8(const float *in, float *out) {
    static const DctBasis basis;  // thread-safe initialisation
    const float(*c)[8] = basis.c;
    float tmp[64];
    for (int y = 0; y < 8; y++)
        for (int k = 0; k < 8; k++) {
            float s = 0;
            for (int x = 0; x < 8; x++) s += c[k][x] * in[8 * y + x];
            tmp[8 * y + k] = s;
        }
    for (int k = 0; k < 8; k++)
        for (int l = 0; l < 8; l++) {
            float s = 0;
            for (int y = 0; y < 8; y++) s += c[l][y] * tmp[8 * y + k];
            out[8 * l + k] = s;
        }
}

inline int bitsize(int v) {
    v = v < 0 ? -v : v;
    int s = 0;
    while (v) {
        s++;
        v >>= 1;
    }
    return s;
}

void put16(std::vector<uint8_t> &o, int v) {
    o.push_back((uint8_t)(v >> 8));
    o.push_back((uint8_t)v);
}

}  // namespace

// flags: 1 = one scan per component (non-interleaved), 2 = SOF1 (extended sequential) frame header, 4 = 16-bit DQT entries,
//        8 = every component on Huffman table 0 (the layout of the reference encoder without colour transformation)
extern "C" __attribute__((visibility("default"))) long b200jpg_synth_encode_ex(const uint8_t *pix, int w, int h, int ncomp, int hs, int vs,
                                                                                 int quality, int dri, int flags, uint8_t *dst, long cap);
extern "C" __attribute__((visibility("default"))) long b200jpg_synth_encode(const uint8_t *pix, int w, int h, int ncomp, int hs, int vs,
                                                                              int quality, int dri, uint8_t *dst, long cap) {
    return b200jpg_synth_encode_ex(pix, w, h, ncomp, hs, vs, quality, dri, 0, dst, cap);
}

extern "C" __attribute__((visibility("default"))) long b200jpg_synth_encode_ex(const uint8_t *pix, int w, int h, int ncomp, int hs, int vs,
                                                                                 int quality, int dri, int flags, uint8_t *dst, long cap) {
    if (!pix || w <= 0 || h <= 0 || (ncomp != 1 && ncomp != 3) || hs < 1 || hs > 2 || vs < 1 || vs > 2) return -1;
    if (ncomp == 1) hs = vs = 1;
    if (quality < 1) quality = 1;
    if (quality > 100) quality = 100;
    int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
    uint8_t q[2][64];
    for (int t = 0; t < 2; t++)
        for (int i = 0; i < 64; i++) {
            int d = ((t ? kChromaQ[i] : kLumaQ[i]) * scale + 50) / 100;
            q[t][i] = (uint8_t)(d < 1 ? 1 : (d > 255 ? 255 : d));
        }
    // planes (level shifted floats), padded to whole MCUs by edge replication
    int mcuw = 8 * hs, mcuh = 8 * vs;
    int mcols = (w + mcuw - 1) / mcuw, mrows = (h + mcuh - 1) / mcuh;
    int pw = mcols * mcuw, ph = mrows * mcuh;
    std::vector<float> Y((size_t)pw * ph), Cb, Cr;
    int cw = pw / hs, chh = ph / vs;
    if (ncomp == 3) {
        Cb.assign((size_t)cw * chh, 0.f);
        Cr.assign((size_t)cw * chh, 0.f);
    }
    std::vector<float> fcb, fcr;
    if (ncomp == 3) {
        fcb.resize((size_t)pw * ph);
        fcr.resize((size_t)pw * ph);
    }
    for (int y = 0; y < ph; y++) {
        int sy = y < h ? y : h - 1;
        for (int x = 0; x < pw; x++) {
            int sx = x < w ? x : w - 1;
            const uint8_t *p = pix + ((size_t)sy * w + sx) * ncomp;
            if (ncomp == 1) {
                Y[(size_t)y * pw + x] = p[0] - 128.f;
            } else {
                float r = p[0], g = p[1], b = p[2];
                Y[(size_t)y * pw + x] = 0.299f * r + 0.587f * g + 0.114f * b - 128.f;
                fcb[(size_t)y * pw + x] = -0.168736f * r - 0.331264f * g + 0.5f * b;
                fcr[(size_t)y * pw + x] = 0.5f * r - 0.418688f * g - 0.081312f * b;
            }
        }
    }
    if (ncomp == 3) {
        for (int y = 0; y < chh; y++)
            for (int x = 0; x < cw; x++) {
                float a = 0, b = 0;
                for (int dy = 0; dy < vs; dy++)
                    for (int dx = 0; dx < hs; dx++) {
                        a += fcb[(size_t)(y * vs + dy) * pw + x * hs + dx];
                        b += fcr[(size_t)(y * vs + dy) * pw + x * hs + dx];
                    }
                Cb[(size_t)y * cw + x] = a / (hs * vs);
                Cr[(size_t)y * cw + x] = b / (hs * vs);
            }
    }
    std::vector<uint8_t> o;
    o.reserve((size_t)w * h / 2 + 4096);
    // headers
    o.push_back(0xff), o.push_back(0xd8);
    const uint8_t jfif[] = {0xff, 0xe0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 2, 0, 0, 1, 0, 1, 0, 0};
    o.insert(o.end(), jfif, jfif + sizeof(jfif));
    const bool wide_q = (flags & 4) != 0;
    o.push_back(0xff), o.push_back(0xdb);
    put16(o, 2 + (ncomp == 3 ? 2 : 1) * (wide_q ? 129 : 65));
    for (int t = 0; t < (ncomp == 3 ? 2 : 1); t++) {
        o.push_back((uint8_t)(t | (wide_q ? 0x10 : 0)));
        for (int i = 0; i < 64; i++) {
            if (wide_q) o.push_back(0);
            o.push_back(q[t][kZZ[i]]);
        }
    }
    if (dri > 0) {
        o.push_back(0xff), o.push_back(0xdd);
        put16(o, 4);
        put16(o, dri);
    }
    o.push_back(0xff), o.push_back((flags & 2) ? 0xc1 : 0xc0);
    put16(o, 8 + 3 * ncomp);
    o.push_back(8);
    put16(o, h);
    put16(o, w);
    o.push_back((uint8_t)ncomp);
    for (int c = 0; c < ncomp; c++) {
        o.push_back((uint8_t)c);
        o.push_back(c == 0 ? (uint8_t)((hs << 4) | vs) : 0x11);
        o.push_back(c == 0 ? 0 : 1);
    }
    o.push_back(0xff), o.push_back(0xc4);
    {
        int len = 2;
        len += 17 + 12 + 17 + 162;
        if (ncomp == 3) len += 17 + 12 + 17 + 162;
        put16(o, len);
        auto tab = [&](int tcth, const uint8_t *bits, const uint8_t *vals, int n) {
            o.push_back((uint8_t)tcth);
            o.insert(o.end(), bits, bits + 16);
            o.insert(o.end(), vals, vals + n);
        };
        tab(0x00, kDcLumBits, kDcVals, 12);
        if (ncomp == 3) tab(0x01, kDcChrBits, kDcVals, 12);
        tab(0x10, kAcLumBits, kAcLumVals, 162);
        if (ncomp == 3) tab(0x11, kAcChrBits, kAcChrVals, 162);
    }
    HuffEnc dcl, dcc, acl, acc_;
    dcl.build(kDcLumBits, kDcVals);
    dcc.build(kDcChrBits, kDcVals);
    acl.build(kAcLumBits, kAcLumVals);
    acc_.build(kAcChrBits, kAcChrVals);
    BitWriter bw(o);
    int pred[3] = {0, 0, 0};
    int togo = dri, rst = 0;
    auto encode_block = [&](const float *plane, int pitch, int bx, int by, int c) {
        float in[64], co[64];
        for (int y = 0; y < 8; y++)
            for (int x = 0; x < 8; x++) in[8 * y + x] = plane[(size_t)(8 * by + y) * pitch + 8 * bx + x];
        fdct8x8(in, co);
        int qc[64];
        const uint8_t *qt = q[c ? 1 : 0];
        for (int i = 0; i < 64; i++) qc[i] = (int)std::lrintf(co[i] / qt[i]);
        const bool chroma_tables = c && !(flags & 8);
        const HuffEnc &dc = chroma_tables ? dcc : dcl, &ac = chroma_tables ? acc_ : acl;
        int diff = qc[0] - pred[c];
        pred[c] = qc[0];
        int s = bitsize(diff);
        bw.put(dc.code[s], dc.len[s]);
        if (s) bw.put((uint32_t)(diff < 0 ? diff - 1 : diff), s);
        int run = 0;
        for (int k = 1; k < 64; k++) {
            int v = qc[kZZ[k]];
            if (v == 0) {
                run++;
                continue;
            }
            while (run > 15) {
                bw.put(ac.code[0xf0], ac.len[0xf0]);
                run -= 16;
            }
            if (v > 1023) v = 1023;
            if (v < -1023) v = -1023;
            s = bitsize(v);
            bw.put(ac.code[(run << 4) | s], ac.len[(run << 4) | s]);
            bw.put((uint32_t)(v < 0 ? v - 1 : v), s);
            run = 0;
        }
        if (run) bw.put(ac.code[0], ac.len[0]);
    };
    auto restart_check = [&]() {
        if (dri > 0) {
            if (togo == 0) {
                bw.flush();
                o.push_back(0xff), o.push_back((uint8_t)(0xd0 + rst));
                rst = (rst + 1) & 7;
                pred[0] = pred[1] = pred[2] = 0;
                togo = dri;
            }
            togo--;
        }
    };
    auto sos = [&](int first, int count) {
        o.push_back(0xff), o.push_back(0xda);
        put16(o, 6 + 2 * count);
        o.push_back((uint8_t)count);
        for (int c = first; c < first + count; c++) {
            o.push_back((uint8_t)c);
            o.push_back(c == 0 || (flags & 8) ? 0x00 : 0x11);
        }
        o.push_back(0), o.push_back(63), o.push_back(0);
        pred[0] = pred[1] = pred[2] = 0;
        togo = dri;
        rst = 0;
    };
    if (!(flags & 1) || ncomp == 1) {  // one interleaved scan
        sos(0, ncomp);
        for (int my = 0; my < mrows; my++)
            for (int mx = 0; mx < mcols; mx++) {
                restart_check();
                for (int y = 0; y < vs; y++)
                    for (int x = 0; x < hs; x++) encode_block(Y.data(), pw, mx * hs + x, my * vs + y, 0);
                if (ncomp == 3) {
                    encode_block(Cb.data(), cw, mx, my, 1);
                    encode_block(Cr.data(), cw, mx, my, 2);
                }
            }
        bw.flush();
    } else {  // one scan per component: the MCU is a single block over the component's own (unpadded) block grid
        for (int c = 0; c < 3; c++) {
            const int compw = c ? (w + hs - 1) / hs : w, comph = c ? (h + vs - 1) / vs : h;
            const int bwc = (compw + 7) / 8, bhc = (comph + 7) / 8;
            sos(c, 1);
            for (int by = 0; by < bhc; by++)
                for (int bx = 0; bx < bwc; bx++) {
                    restart_check();
                    encode_block(c == 0 ? Y.data() : (c == 1 ? Cb.data() : Cr.data()), c ? cw : pw, bx, by, c);
                }
            bw.flush();
        }
    }
    o.push_back(0xff), o.push_back(0xd9);
    if ((long)o.size() > cap || !dst) return -(long)o.size();
    memcpy(dst, o.data(), o.size());
    return (long)o.size();
}
