// progressive_sm100.cu -- SURVEY 8f2: progressive (SOF2) Huffman scans on sm_90a.
//
// Replaces, for progressive frames, the reference's
//   SequentialScan::DecodeBlock with m_bProgressive     codestream/sequentialscan.cpp:678-773 (DC / AC first passes:
//                                                       EOB runs :722-726, point transform `<< lowbit`)
//   RefinementScan::DecodeBlock                         codestream/refinementscan.cpp:584-690 (DC refinement: one raw bit
//                                                       per block :588-592; AC refinement: correction bits :616-626)
//   SequentialScan::Restart / RefinementScan::Restart   (DC predictors and EOB run reset per restart interval)
//
// Work decomposition is the one of the sequential entropy kernel -- a restart interval is an independent bit stream, one per
// lane, fed from the unstuffed big-endian words that unstuff_kernel (a0) produced -- but the scans of a frame build on each
// other, so every scan class is one launch, in scan order, and the coefficient store (int16, 128 bytes per block, raster
// order) holds QUANTISED levels that the passes read and update in place. progressive_dequant_kernel turns them into the
// dequantised coefficients stage b expects once the last scan is done.  This is the first, straightforward version of the
// path (lanes walk their blocks independently, coefficients are read and written in HBM through L1/L2 without staging): it
// is parity-complete, not tuned.
#include <cuda_runtime.h>

#include <cstdint>

#include "internal.hpp"

namespace b200jpg {
namespace {

constexpr int kThreadsP = 256;
constexpr uint32_t kErrMalformed = 1038u;      // -(-1038) MALFORMED_STREAM
constexpr uint32_t kErrUnexpectedEof = 1025u;  // -(-1025) UNEXPECTED_EOF

__constant__ uint8_t c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};  // dct/dct.cpp:57-73

// Bit reader over the unstuffed words of one interval: bit position + the three words around it, like the sequential
// kernel's, but the words come straight from HBM (L1-cached); past the end it hands out zeros, which is what the
// reference's reader does once it stands in front of a marker (io/bitstream.cpp:96-101).
struct Bits {
    const uint32_t *w;
    uint32_t nwords, bp, xw, x0, x1, x2;
    __device__ __forceinline__ uint32_t word(uint32_t i) const { return i < nwords ? __ldg(w + i) : 0u; }
    __device__ __forceinline__ void open(const uint8_t *p, uint32_t len_bytes) {
        w = reinterpret_cast<const uint32_t *>(p);
        nwords = (len_bytes + 3u) / 4u;
        bp = 0, xw = 0;
        x0 = word(0), x1 = word(1), x2 = word(2);
    }
    __device__ __forceinline__ uint32_t window() const { return __funnelshift_l(x1, x0, bp); }
    __device__ __forceinline__ void skip(uint32_t n) {  // n < 32
        bp += n;
        const uint32_t wi = bp >> 5;
        if (wi != xw) {
            x0 = x1, x1 = x2, x2 = word(wi + 2u), xw = wi;
        }
    }
    __device__ __forceinline__ uint32_t get(uint32_t n) {  // n <= 16
        const uint32_t v = n ? (window() >> (32u - n)) : 0u;
        skip(n);
        return v;
    }
};

// one Huffman symbol: returns the table entry (fields: internal.hpp; progressive flavour keeps the raw run in [13:10])
__device__ __forceinline__ uint32_t symbol(Bits &b, const uint32_t *lut) {
    const uint32_t hi = b.window();
    uint32_t e = lut[hi >> (32 - kLutL1Bits)];
    if ((e & (31u << 5)) == 0) e = lut[(1u << kLutL1Bits) + ((e >> 10) << (16 - kLutL1Bits)) + ((hi >> 16) & ((1u << (16 - kLutL1Bits)) - 1u))];
    b.skip((e >> 5) & 31u);
    return e;
}

__device__ __forceinline__ int extend(uint32_t v, uint32_t s) {  // sequentialscan.cpp:692-696 / 757-762
    return (v < (1u << (s - 1))) ? (int)v + (int)((~0u) << s) + 1 : (int)v;
}

__global__ void __launch_bounds__(kThreadsP)
progressive_scan_kernel(ScanClassParams p, const uint8_t *__restrict__ clean, const uint64_t *__restrict__ clean_off,
                        const uint32_t *__restrict__ interval_len, const ClassScan *__restrict__ scans, const uint8_t *__restrict__ tables,
                        int16_t *__restrict__ coef, uint32_t *__restrict__ frame_status) {
    extern __shared__ uint32_t s_lut[];
    const uint32_t *g_lut = reinterpret_cast<const uint32_t *>(tables + kTableHeaderBytes);
    for (uint32_t i = threadIdx.x; i < p.lut_words; i += kThreadsP) s_lut[i] = g_lut[i];
    __syncthreads();
    const uint16_t *lut_off = reinterpret_cast<const uint16_t *>(tables + 16);

    const uint64_t total_intervals = (uint64_t)p.n_scans * p.intervals_per_scan;
    const uint64_t g = (uint64_t)blockIdx.x * kThreadsP + threadIdx.x;
    if (g >= total_intervals) return;
    const uint32_t j = (uint32_t)(g / p.intervals_per_scan), iv = (uint32_t)(g % p.intervals_per_scan);
    const uint32_t len_raw = interval_len[g];
    const uint32_t len_bytes = len_raw & kIntervalLenMask;
    if (len_raw & kIntervalLenAbsent) return;  // an interval the stream does not contain leaves its blocks as they are
    const ClassScan &cs = scans[j];
    const uint32_t mcu0 = iv * p.dri;
    const uint32_t nmcu = (p.total_mcus - mcu0 < p.dri) ? (p.total_mcus - mcu0) : p.dri;
    uint32_t mx = mcu0 % p.mcu_cols, my = mcu0 / p.mcu_cols;

    Bits b;
    b.open(clean + clean_off[g], len_bytes);
    int pred[4] = {0, 0, 0, 0};
    uint32_t skip = 0;  // blocks an EOB run still covers (AC scans carry one component)
    bool bad = false;
    const int al = p.al;
    const bool first = p.ah == 0;

    for (uint32_t mi = 0; mi < nmcu && !bad; mi++) {
        for (int c = 0; c < p.ns && !bad; c++) {
            const uint32_t *dc = s_lut + ((p.ss == 0 && first) ? lut_off[p.dc_slot[c]] : 0);
            const uint32_t *ac = s_lut + ((p.se != 0) ? lut_off[4 + p.ac_slot[c]] : 0);
            for (int y = 0; y < p.mh[c] && !bad; y++) {
                for (int x = 0; x < p.mw[c] && !bad; x++) {
                    const uint32_t bx = mx * p.mw[c] + x, by = my * p.mh[c] + y;
                    int16_t *blk = coef + cs.coef_base[c] + ((uint64_t)by * p.bw[c] + bx) * 64u;
                    if (p.ss == 0) {
                        if (first) {  // DC, first pass: sequentialscan.cpp:682-701
                            const uint32_t e = symbol(b, dc);
                            if ((int)e < 0) {
                                bad = true;
                                break;
                            }
                            const uint32_t s = e & 31u;
                            if (s) pred[c] += extend(b.get(s), s);
                            blk[0] = (int16_t)((uint32_t)pred[c] << al);
                        } else {      // DC refinement: one raw bit, refinementscan.cpp:588-592
                            blk[0] = (int16_t)(blk[0] | (int)(b.get(1) << al));
                        }
                        continue;
                    }
                    if (first) {      // AC, first pass: sequentialscan.cpp:704-772
                        if (skip > 0) {
                            skip--;
                            continue;
                        }
                        int k = p.ss;
                        do {
                            const uint32_t e = symbol(b, ac);
                            if ((int)e < 0) {
                                bad = true;
                                break;
                            }
                            const uint32_t r = (e >> 10) & 15u, s = e & 31u;
                            if (s == 0) {
                                if (r == 15) {
                                    k += 16;
                                    continue;
                                }
                                skip = (1u << r) | b.get(r);  // EOBn
                                skip--;                       // this block is part of the run
                                break;
                            }
                            k += (int)r;
                            const int v = extend(b.get(s), s);
                            if (k >= 64) {  // the reference tests against 64, not against Se
                                bad = true;
                                break;
                            }
                            blk[c_zigzag[k]] = (int16_t)((uint32_t)v << al);
                            k++;
                        } while (k <= p.se);
                    } else {          // AC refinement: refinementscan.cpp:594-690
                        int k = p.ss;
                        if (skip == 0) {
                            while (k <= p.se) {
                                const uint32_t e = symbol(b, ac);
                                if ((int)e < 0) {
                                    bad = true;
                                    break;
                                }
                                uint32_t r = (e >> 10) & 15u;
                                const uint32_t s = e & 31u;
                                int val = 0;
                                if (s == 0) {
                                    if (r != 15) {  // EOBn: the rest of the block only takes correction bits
                                        skip = (1u << r) | b.get(r);
                                        break;
                                    }
                                } else if (s != 1) {  // the reference warns and goes on with a zero amplitude (:659-668)
                                    r = 0;
                                } else {
                                    val = b.get(1) ? (1 << al) : -(1 << al);
                                }
                                while (k <= p.se) {  // pass r zero-valued positions; significant ones take a correction bit
                                    int16_t *q = blk + c_zigzag[k];
                                    const int cur = *q;
                                    if (cur) {
                                        if (b.get(1)) *q = (int16_t)(cur + (cur > 0 ? (1 << al) : -(1 << al)));
                                    } else {
                                        if (r == 0) break;
                                        r--;
                                    }
                                    k++;
                                }
                                if (k <= p.se) blk[c_zigzag[k]] = (int16_t)val;  // the zero-valued position that ends the run
                                k++;
                            }
                        }
                        if (skip > 0 && !bad) {
                            for (; k <= p.se; k++) {
                                int16_t *q = blk + c_zigzag[k];
                                const int cur = *q;
                                if (cur && b.get(1)) *q = (int16_t)(cur + (cur > 0 ? (1 << al) : -(1 << al)));
                            }
                            skip--;
                        }
                    }
                }
            }
        }
        if (++mx == p.mcu_cols) {
            mx = 0;
            my++;
        }
    }
    uint32_t err = 0;
    if (bad) err = kErrMalformed;
    else if ((uint64_t)b.bp > (uint64_t)len_bytes * 8u && !(len_raw & kIntervalLenEofFlag)) err = kErrUnexpectedEof;  // consumed bits beyond the interval's marker
    if (err) atomicMax(frame_status + cs.frame, err);
}

// quantised level x quantiser -> the int16 coefficient stage b reads (the IDCT applies the remaining << 4, dct/idct.cpp:98-108)
__global__ void __launch_bounds__(256)
progressive_dequant_kernel(const ProgFrame *__restrict__ frames, int16_t *__restrict__ coef, uint32_t *__restrict__ frame_status) {
    const ProgFrame &f = frames[blockIdx.y];
    const int c = blockIdx.z;
    const uint32_t t = blockIdx.x * 256u + threadIdx.x;  // one 8-coefficient row of a block per thread
    if (t >= f.n_blocks[c] * 8u) return;
    uint4 *p = reinterpret_cast<uint4 *>(coef + f.coef_base[c]) + t;
    uint4 v = *p;
    const uint16_t *q = f.q_raster[c] + 8u * (t & 7u);
    uint32_t ovf = 0;
    uint32_t *w = &v.x;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int lo = (int)(short)(w[i] & 0xffffu) * (int)q[2 * i], hi = ((int)w[i] >> 16) * (int)q[2 * i + 1];
        ovf |= (uint32_t)(lo + 32768) | (uint32_t)(hi + 32768);
        w[i] = ((uint32_t)lo & 0xffffu) | ((uint32_t)hi << 16);
    }
    *p = v;
    if (ovf >> 16) atomicMax(frame_status + f.frame, kErrMalformed);  // a coefficient beyond the int16 store
}

}  // namespace

int launch_progressive_scan(const EntropyLaunch &l, void *stream) {
    const uint64_t total = (uint64_t)l.p.n_scans * l.p.intervals_per_scan;
    if (total == 0) return 0;
    const size_t smem = (size_t)l.p.lut_words * 4;
    cudaError_t e;
    if (smem > 48 * 1024) {
        e = cudaFuncSetAttribute(progressive_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    const uint32_t grid = (uint32_t)((total + kThreadsP - 1) / kThreadsP);
    progressive_scan_kernel<<<grid, kThreadsP, smem, (cudaStream_t)stream>>>(l.p, l.clean, l.clean_off, l.interval_len, l.scans, l.tables, l.coef,
                                                                              l.frame_status);
    return (int)cudaGetLastError();
}

int launch_progressive_dequant(const ProgFrame *frames_dev, uint32_t n_frames, uint32_t max_blocks, int16_t *coef, uint32_t *frame_status,
                               void *stream) {
    if (n_frames == 0 || max_blocks == 0) return 0;
    for (uint32_t first = 0; first < n_frames; first += 65535u) {  // grid.y carries the frame index
        const uint32_t part = n_frames - first < 65535u ? n_frames - first : 65535u;
        dim3 grid((max_blocks * 8u + 255u) / 256u, part, 4);
        progressive_dequant_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(frames_dev + first, coef, frame_status);
    }
    return (int)cudaGetLastError();
}

}  // namespace b200jpg
