// recon_sm100.cu -- stage (b): integer IDCT + centred-bilinear chroma upsampling + YCbCr->RGB + 8-bit store.
//
// Replaces the reference's reconstruction path (bit-exact, all int32 like the reference's LONG):
//   BlockBitmapRequester::ReconstructRegion / PullQData / PushReconstructedData / ReconstructUnsampled
//                                                     control/blockbitmaprequester.cpp:1249-1272,1079-1112,1151-1224,1013-1074
//   IDCT<4,LONG,false,false>::InverseTransformBlock   dct/idct.cpp:226-339 (constants idct.cpp:65-78, idct.hpp:70-77)
//   UpsamplerBase::DefineRegion (edge replication)    upsampling/upsamplerbase.cpp:300-327
//   Upsampler<sx,sy>::UpsampleRegion                  upsampling/upsampler.cpp:83-112
//   VerticalFilterCore<1|2>, HorizontalFilterCore<1|2> upsampling/upsampler.cpp:114-168, 270-307 (incl. the in-place
//                                                     read-after-write of out[1], :301-302, which is part of the contract)
//   YCbCrTrafo<UBYTE,3,ClampFlag,YCbCr,Zero>::YCbCr2RGB colortrafo/ycbcrtrafo.cpp:679-1008 (:842-850, :922-935)
//
// Mapping.  One thread owns one 8x8 block.
//  4:2:0 frames: reconstruct420_kernel, one kernel from coefficients to pixels (chroma IDCT into a shared-memory window,
//     then the luma rows exactly like b2); see its section below.  Every other 1..3 component format:
//  b1 idct_planes_kernel: blocks of the non-luma components -> int32 sample planes (the whole-frame equivalent of
//     the reference's upsampler line buffers); both 1-D passes in registers.
//  b2 reconstruct_kernel: a warp owns 32 horizontally adjacent luma blocks (256 x 8 pixels), a CTA four such rows.
//     The warp's 4 KB of coefficients come in with coalesced 16-byte loads and are handed to their lanes through
//     shared memory; the row pass and the column pass of the luma IDCT run as two compact loops over a shared-memory
//     tile laid out [coefficient][thread] (bank-conflict free, thread-private columns); a third loop walks the eight
//     output lines: chroma window from the planes (clamped addressing = the reference's edge replication at the true
//     subsampled size), vertical + horizontal filter cores, colour transform, and each lane stores its 24 bytes of
//     interleaved RGB per line.  The kernel is co-limited by instruction issue and by the L1 data pipe, so global
//     accesses are shaped for few L1 wavefronts; small loop bodies keep it inside the instruction cache (the fully
//     unrolled register-resident version stalled on instruction fetch).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <type_traits>

#include "cmyk_sm90.cuh"
#include "internal.hpp"
#include "store_sm90.cuh"

namespace b200jpg {
namespace {

constexpr int kWide = 65535;  // |sample| above this may overflow the 32-bit colour arithmetic -> 64-bit path

#define WMUL(a, k) ((int)((unsigned)(a) * (unsigned)(int)(k)))
#define WADD(a, b) ((int)((unsigned)(a) + (unsigned)(b)))
#define WSUB(a, b) ((int)((unsigned)(a) - (unsigned)(b)))

// One 8-point pass of dct/idct.cpp:237-287 (rows, round = 256, shift = 9) / :291-334 (columns, 2048, 12).
// Constants are WORD(x * 512 + 0.5) of the reference's TO_FIX table.
template <int kRound, int kShift>
__device__ __forceinline__ void idct8(int &v0, int &v1, int &v2, int &v3, int &v4, int &v5, int &v6, int &v7) {
    int z1 = WMUL(WADD(v2, v6), 277);
    int tmp2 = WADD(z1, WMUL(v6, -946));
    int tmp3 = WADD(z1, WMUL(v2, 392));
    int tmp0 = (int)((unsigned)WADD(v0, v4) << 9);
    int tmp1 = (int)((unsigned)WSUB(v0, v4) << 9);
    int tmp10 = WADD(tmp0, tmp3), tmp13 = WSUB(tmp0, tmp3);
    int tmp11 = WADD(tmp1, tmp2), tmp12 = WSUB(tmp1, tmp2);
    int t0 = v7, t1 = v5, t2 = v3, t3 = v1;
    int y1 = WADD(t0, t3), y2 = WADD(t1, t2), y3 = WADD(t0, t2), y4 = WADD(t1, t3);
    int z5 = WMUL(WADD(y3, y4), 602);
    t0 = WMUL(t0, 153);
    t1 = WMUL(t1, 1051);
    t2 = WMUL(t2, 1573);
    t3 = WMUL(t3, 769);
    y1 = WMUL(y1, -461);
    y2 = WMUL(y2, -1312);
    y3 = WADD(WMUL(y3, -1004), z5);
    y4 = WADD(WMUL(y4, -200), z5);
    t0 = WADD(t0, WADD(y1, y3));
    t1 = WADD(t1, WADD(y2, y4));
    t2 = WADD(t2, WADD(y2, y3));
    t3 = WADD(t3, WADD(y1, y4));
    v0 = WADD(WADD(tmp10, t3), kRound) >> kShift;
    v7 = WADD(WSUB(tmp10, t3), kRound) >> kShift;
    v1 = WADD(WADD(tmp11, t2), kRound) >> kShift;
    v6 = WADD(WSUB(tmp11, t2), kRound) >> kShift;
    v2 = WADD(WADD(tmp12, t1), kRound) >> kShift;
    v5 = WADD(WSUB(tmp12, t1), kRound) >> kShift;
    v3 = WADD(WADD(tmp13, t0), kRound) >> kShift;
    v4 = WADD(WSUB(tmp13, t0), kRound) >> kShift;
}

// eight dequantised int16 coefficients (one block row) -> ints carrying the << 4 preshift of dct/idct.cpp:105
__device__ __forceinline__ void unpack_row(const uint4 q, int (&v)[8]) {
    v[0] = (int)(short)(q.x & 0xffffu) << 4;
    v[1] = (int)(short)(q.x >> 16) << 4;
    v[2] = (int)(short)(q.y & 0xffffu) << 4;
    v[3] = (int)(short)(q.y >> 16) << 4;
    v[4] = (int)(short)(q.z & 0xffffu) << 4;
    v[5] = (int)(short)(q.z >> 16) << 4;
    v[6] = (int)(short)(q.w & 0xffffu) << 4;
    v[7] = (int)(short)(q.w >> 16) << 4;
}

// ---- instruction-selection helpers ---------------------------------------------------------------------------------------
// Both integer pipes of an SM sub-partition (ALU: IADD3 / SHF / LOP3 / LEA / PRMT; FMA-heavy: IMAD, IMAD.IADD, IMAD.MOV, VIADD)
// take one warp instruction every other cycle (tools/opbench.cu), so the kernel runs at the pace of the fuller one. ptxas likes "x * 3 + y" as IMAD followed by VIADD for the rounding constant: two
// FMA-heavy instructions per filter tap. Spelled as below it emits IADD3 (a + b + r) and one IMAD (b * 2 + t): one on each pipe.
#ifndef B200JPG_FUSED_PLAIN
__device__ __forceinline__ int add3(int a, int b, int c) {
    int d;
    asm("{ .reg .s32 x; add.s32 x, %1, %2; add.s32 %0, x, %3; }" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
template <int C>
__device__ __forceinline__ int add2c(int a, int b) {  // a + b + C
    int d;
    asm("{ .reg .s32 x; add.s32 x, %1, %2; add.s32 %0, x, %3; }" : "=r"(d) : "r"(a), "r"(b), "n"(C));
    return d;
}
template <int C>
__device__ __forceinline__ int sub2c(int a, int b) {  // a - b + C
    int d;
    asm("{ .reg .s32 x; sub.s32 x, %1, %2; add.s32 %0, x, %3; }" : "=r"(d) : "r"(a), "r"(b), "n"(C));
    return d;
}
// (a + 3 b + R) >> 2: upsampling/upsampler.cpp:136-168, 283-307
template <int R>
__device__ __forceinline__ int tap(int a, int b) {
    int d;
    asm("{ .reg .s32 x, y; add.s32 x, %1, %2; add.s32 x, x, %3; shl.b32 y, %2, 1; add.s32 x, x, y; shr.s32 %0, x, 2; }" : "=r"(d) : "r"(a), "r"(b), "n"(R));
    return d;
}
#else
__device__ __forceinline__ int add3(int a, int b, int c) { return WADD(WADD(a, b), c); }
template <int C>
__device__ __forceinline__ int add2c(int a, int b) { return WADD(WADD(a, b), C); }
template <int C>
__device__ __forceinline__ int sub2c(int a, int b) { return WADD(WSUB(a, b), C); }
template <int R>
__device__ __forceinline__ int tap(int a, int b) { return WADD(WADD(a, WMUL(3, b)), R) >> 2; }
#endif

// HorizontalFilterCore<2> (upsampler.cpp:283-307) on w[0..5] with the taps above
__device__ __forceinline__ void hfilter2t(const int (&w)[6], int (&o)[8]) {
    o[7] = tap<1>(w[5], w[4]);
    o[6] = tap<2>(w[3], w[4]);
    o[5] = tap<1>(w[4], w[3]);
    o[4] = tap<2>(w[2], w[3]);
    o[3] = tap<1>(w[3], w[2]);
    o[2] = tap<2>(w[1], w[2]);
    o[1] = tap<1>(o[2], w[1]);  // reads the freshly written out[2] (upsampler.cpp:301-302)
    o[0] = tap<2>(w[0], w[1]);
}

// One 8-point pass like idct8, with the rounding constant riding in the three-input adds of the outputs
template <int kRound, int kShift>
__device__ __forceinline__ void idct8t(int &v0, int &v1, int &v2, int &v3, int &v4, int &v5, int &v6, int &v7) {
    const int z1 = WMUL(WADD(v2, v6), 277);
    const int tmp2 = WADD(z1, WMUL(v6, -946));
    const int tmp3 = WADD(z1, WMUL(v2, 392));
    const int a04 = WADD(v0, v4), s04 = WSUB(v0, v4);
    const int tmp10 = WADD(WMUL(a04, 512), tmp3), tmp13 = WSUB(WMUL(a04, 512), tmp3);
    const int tmp11 = WADD(WMUL(s04, 512), tmp2), tmp12 = WSUB(WMUL(s04, 512), tmp2);
    const int y1 = WADD(v7, v1), y2 = WADD(v5, v3), y3 = WADD(v7, v3), y4 = WADD(v5, v1);
    const int z5 = WMUL(WADD(y3, y4), 602);
    const int p1 = WMUL(y1, -461), p2 = WMUL(y2, -1312);
    const int p3 = WADD(WMUL(y3, -1004), z5), p4 = WADD(WMUL(y4, -200), z5);
    const int t0 = WADD(WADD(WMUL(v7, 153), p1), p3);
    const int t1 = WADD(WADD(WMUL(v5, 1051), p2), p4);
    const int t2 = WADD(WADD(WMUL(v3, 1573), p2), p3);
    const int t3 = WADD(WADD(WMUL(v1, 769), p1), p4);
    v0 = add2c<kRound>(tmp10, t3) >> kShift;
    v7 = sub2c<kRound>(tmp10, t3) >> kShift;
    v1 = add2c<kRound>(tmp11, t2) >> kShift;
    v6 = sub2c<kRound>(tmp11, t2) >> kShift;
    v2 = add2c<kRound>(tmp12, t1) >> kShift;
    v5 = sub2c<kRound>(tmp12, t1) >> kShift;
    v3 = add2c<kRound>(tmp13, t0) >> kShift;
    v4 = sub2c<kRound>(tmp13, t0) >> kShift;
}

// eight dequantised int16 coefficients -> ints WITHOUT the << 4 preshift of dct/idct.cpp:105. The row pass is linear in front
// of its rounding shift, so with inputs 16 times smaller ((16 x + 256) >> 9) == ((x + 16) >> 5) for every integer x. The
// reference's int32 arithmetic cannot wrap in this pass: the absolute weights of every output sum to 3825 (the DC's is 512),
// so for coefficients within +-32767 no sum exceeds 16 (3825 * 32767 + 512 * (dcoffset << 3)) + 256, which is 2,013,729,264
// for 8 bit (dcoffset << 3 = 1024) and 2,139,558,384 for 12 bit (16384); a row of DC 32767 and ACs of 32767 with the signs of
// one output's weights reaches it (tests/recon_cases.py, rowmax_8 / rowmax_12). A dequantised -32768 where a weight is
// negative adds at most 16 * 2434: 2,013,768,208 and 2,139,597,328 (0.4 % below 2^31). So nothing is lost by never forming
// 16 x.
__device__ __forceinline__ void unpack_row_raw(const uint4 q, int (&v)[8]) {
    v[0] = (int)(short)(q.x & 0xffffu);
    v[1] = (int)q.x >> 16;
    v[2] = (int)(short)(q.y & 0xffffu);
    v[3] = (int)q.y >> 16;
    v[4] = (int)(short)(q.z & 0xffffu);
    v[5] = (int)q.z >> 16;
    v[6] = (int)(short)(q.w & 0xffffu);
    v[7] = (int)q.w >> 16;
}

// ---- b1: non-luma components -> sample planes ---------------------------------------------------------
// Samples of real images fit 16 bits with room to spare, so the planes that every frame goes through are int16
// (half the HBM traffic of this memory-bound kernel). A frame in which any sample does not fit is flagged `narrow`
// and redone by the same kernels instantiated for int32 planes (kListed: they walk the list of flagged frames
// instead of the whole group, so the exact pass costs three tiny launches when nothing is flagged).
constexpr int kWideSlots = 4;  // grid extent of the exact pass in the frame dimension; each slot strides over the list

template <typename T>
__device__ __forceinline__ void idct_planes_block(const FrameRecon &f, int c, uint32_t t, const int16_t *__restrict__ coef,
                                                  T *__restrict__ samples, uint32_t *__restrict__ flags) {
    const uint32_t bw = f.bw[c], bh = f.bh[c];
    if (t >= bw * bh) return;
    const uint32_t bx = t % bw, by = t / bw;
    int s[8][8];
    const uint4 *src = reinterpret_cast<const uint4 *>(coef + f.coef_base[c] + (uint64_t)t * 64u);
#pragma unroll
    for (int r = 0; r < 8; r++) unpack_row_raw(__ldg(src + r), s[r]);
    // dcoffset << 3 (idct.cpp:233,244); the << 4 preshift is folded into the row pass' rounding. 12-bit frames only come
    // through the int32 planes (tables.cpp:1877-1891: the same LONG IDCT, level shift 1 << 11)
    s[0][0] = WADD(s[0][0], sizeof(T) == 4 ? (int)(8u << (f.precision - 1u)) : (128 << 3));
#pragma unroll
    for (int r = 0; r < 8; r++) idct8t<16, 5>(s[r][0], s[r][1], s[r][2], s[r][3], s[r][4], s[r][5], s[r][6], s[r][7]);
    int mx = 0, mn = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        idct8t<2048, 12>(s[0][k], s[1][k], s[2][k], s[3][k], s[4][k], s[5][k], s[6][k], s[7][k]);
#pragma unroll
        for (int r = 0; r < 8; r += 2) {
            mx = __vimax3_s32(mx, s[r][k], s[r + 1][k]);
            mn = __vimin3_s32(mn, s[r][k], s[r + 1][k]);
        }
    }
    const uint32_t pitch = 8u * bw;
    T *dst = samples + f.sample_base[c] + (uint64_t)(8u * by) * pitch + 8u * bx;
    if (sizeof(T) == 2) {
        if (mx > 32767 || mn < -32768) atomicOr(flags + f.status_idx, 1u);  // `narrow`: the frame needs the int32 planes
#pragma unroll
        for (int r = 0; r < 8; r++) {
            uint4 w;
            w.x = ((uint32_t)s[r][0] & 0xffffu) | ((uint32_t)s[r][1] << 16);
            w.y = ((uint32_t)s[r][2] & 0xffffu) | ((uint32_t)s[r][3] << 16);
            w.z = ((uint32_t)s[r][4] & 0xffffu) | ((uint32_t)s[r][5] << 16);
            w.w = ((uint32_t)s[r][6] & 0xffffu) | ((uint32_t)s[r][7] << 16);
            *reinterpret_cast<uint4 *>(dst + (uint64_t)r * pitch) = w;
        }
    } else {
        if (mx > kWide || mn < -kWide) atomicOr(flags + f.status_idx, 1u);  // `wide`: colour needs 64 bits
#pragma unroll
        for (int r = 0; r < 8; r++) {
            int4 *d = reinterpret_cast<int4 *>(dst + (uint64_t)r * pitch);
            d[0] = make_int4(s[r][0], s[r][1], s[r][2], s[r][3]);
            d[1] = make_int4(s[r][4], s[r][5], s[r][6], s[r][7]);
        }
    }
}

// grid (blocks / 128, frames or kWideSlots, components - 1); list = {count, frame indices...} for kListed
template <typename T, bool kListed>
__global__ void __launch_bounds__(kThreadsB)
idct_planes_kernel(const FrameRecon *__restrict__ frames, const int16_t *__restrict__ coef, T *__restrict__ samples, uint32_t *__restrict__ flags,
                   const uint32_t *__restrict__ list, int first_comp) {
    const int c = first_comp + blockIdx.z;
    const uint32_t t = blockIdx.x * kThreadsB + threadIdx.x;
    if (!kListed) {
        const FrameRecon &f = frames[blockIdx.y];
        if (c < (int)f.ncomp) idct_planes_block<T>(f, c, t, coef, samples, flags);
    } else {
        const uint32_t n = list[0];
        for (uint32_t k = blockIdx.y; k < n; k += gridDim.y) {
            const FrameRecon &f = frames[list[1 + k]];
            if (c < (int)f.ncomp) idct_planes_block<T>(f, c, t, coef, samples, flags);
        }
    }
}

// idct_planes_kernel for cropped frames: only the chroma blocks [cb_x0, cb_x1) x [cb_y0, cb_y1) that the frame's tiles read;
// grid (range blocks / 128, frames or kWideSlots, components - 1)
template <typename T, bool kListed>
__global__ void __launch_bounds__(kThreadsB)
idct_planes_crop_kernel(const FrameRecon *__restrict__ frames, const int16_t *__restrict__ coef, T *__restrict__ samples, uint32_t *__restrict__ flags,
                        const uint32_t *__restrict__ list, int first_comp) {
    const int c = first_comp + blockIdx.z;
    const uint32_t t = blockIdx.x * kThreadsB + threadIdx.x;
    auto one = [&](const FrameRecon &f) {
        const uint32_t rw = f.cb_x1 - f.cb_x0, rh = f.cb_y1 - f.cb_y0;
        if (c < (int)f.ncomp && t < rw * rh) idct_planes_block<T>(f, c, (f.cb_y0 + t / rw) * f.bw[c] + f.cb_x0 + t % rw, coef, samples, flags);
    };
    if (!kListed) {
        one(frames[blockIdx.y]);
    } else {
        const uint32_t n = list[0];
        for (uint32_t k = blockIdx.y; k < n; k += gridDim.y) one(frames[list[1 + k]]);
    }
}

// ---- downscaled decoding (B200JPG_FLAG_DOWNSCALE_k): blocks -> (8/k) x (8/k) int32 samples -------------------------------
// The k x k box average of the exact 8-point IDCT is, per dimension, the (8/k) x 8 matrix
//     A_k(m, u) = 1/k sum_{j<k} C(u)/2 cos((2 (k m + j) + 1) u pi / 16),   C(0) = 1/sqrt(2), else 1
// (for k = 2 the 4-point IDCT of the folded coefficients; DESIGN §10). With a_k = round(2^20 A_k) and F the dequantised
// coefficients in raster order (row r = vertical frequency), the samples -- 4 fractional bits, level shifted, like the
// planes of idct_planes_kernel -- are, with every sum in int64 (|F| <= 2^15 and sum_u |A_k(m, u)| < 1.69: nothing wraps)
//     row pass     P[r][m] = (sum_u a_k[m][u] F[r][u] + 2^7) >> 8                        |P| < 2^28
//     column pass  s[n][m] = ((sum_r a_k[n][r] P[r][m] + 2^27) >> 28) + (8 << precision)
// and for k = 8, where only the DC term is left, exactly s = 2 F[0][0] + (8 << precision).
__constant__ int kScaledBasis2[4][8] = {{370728, 475072, 342508, 166823, 0, -111468, -141871, -94498},
                                        {370728, 196781, -342508, -402746, 0, 269107, 141871, -39142},
                                        {370728, -196781, -342508, 402746, 0, -269107, 141871, 39142},
                                        {370728, -475072, 342508, -166823, 0, 111468, -141871, 94498}};
__constant__ int kScaledBasis4[2][8] = {{370728, 335926, 0, -117962, 0, 78819, 0, -66820}, {370728, -335926, 0, 117962, 0, -78819, 0, 66820}};

template <int KS>
__device__ __forceinline__ int scaled_basis(int m, int u) {
    return KS == 2 ? kScaledBasis2[m][u] : kScaledBasis4[m][u];
}

// the (8/k) x (8/k) samples of one block (k = 2, 4, 8), level shifted by `level` = 8 << precision; for k = 8 only the block's DC
// word is read
template <int KS>
__device__ __forceinline__ void scaled_idct_block(const int16_t *__restrict__ blk, int level, int (&s)[8 / KS][8 / KS]) {
    constexpr int N = 8 / KS;
    if constexpr (KS == 8) {
        s[0][0] = 2 * (int)__ldg(blk) + level;
    } else {
        const uint4 *src = reinterpret_cast<const uint4 *>(blk);
        int p[8][N];
#pragma unroll
        for (int r = 0; r < 8; r++) {
            int v[8];
            unpack_row_raw(__ldg(src + r), v);
#pragma unroll
            for (int m = 0; m < N; m++) {
                long long acc = 1ll << 7;
#pragma unroll
                for (int u = 0; u < 8; u++) acc += (long long)scaled_basis<KS>(m, u) * v[u];
                p[r][m] = (int)(acc >> 8);
            }
        }
#pragma unroll
        for (int n = 0; n < N; n++) {
#pragma unroll
            for (int m = 0; m < N; m++) {
                long long acc = 1ll << 27;
#pragma unroll
                for (int r = 0; r < 8; r++) acc += (long long)scaled_basis<KS>(n, r) * p[r][m];
                s[n][m] = (int)(acc >> 28) + level;
            }
        }
    }
}

// grid (coefficient blocks / 128, frames, components). Block (bx, by) of the coefficient grid coef_bw x coef_bh lands at
// ((8/k) bx, (8/k) by) of a plane whose FrameRecon grid bw x bh = ceil(coef_bw / k) x ceil(coef_bh / k) makes the pitch
// 8 bw >= (8/k) coef_bw: the generic kernels address the planes of the reduced frame like any other
template <int KS>
__global__ void __launch_bounds__(kThreadsB)
idct_scaled_planes_kernel(const FrameRecon *__restrict__ frames, const int16_t *__restrict__ coef, int32_t *__restrict__ samples) {
    constexpr int N = 8 / KS;
    const FrameRecon &f = frames[blockIdx.y];
    const uint32_t c = blockIdx.z;
    if (c >= f.ncomp) return;
    const uint32_t cbw = f.coef_bw[c], t = blockIdx.x * kThreadsB + threadIdx.x;
    if (t >= cbw * f.coef_bh[c]) return;
    const uint32_t bx = t % cbw, by = t / cbw, pitch = 8u * f.bw[c];
    int s[N][N];
    scaled_idct_block<KS>(coef + f.coef_base[c] + (uint64_t)t * 64u, (int)(8u << f.precision), s);
    int32_t *dst = samples + f.sample_base[c] + (uint64_t)(N * by) * pitch + N * bx;
#pragma unroll
    for (int n = 0; n < N; n++) {
        int32_t *row = dst + (uint64_t)n * pitch;
        if (N == 4) *reinterpret_cast<int4 *>(row) = make_int4(s[n][0], s[n][N > 1 ? 1 : 0], s[n][N > 2 ? 2 : 0], s[n][N > 3 ? 3 : 0]);
        else if (N == 2) *reinterpret_cast<int2 *>(row) = make_int2(s[n][0], s[n][N > 1 ? 1 : 0]);
        else row[0] = s[n][0];
    }
}

// the frames of a group whose `narrow` flag is set -> list = {count, group-local indices}
__global__ void __launch_bounds__(256)
narrow_list_kernel(const FrameRecon *__restrict__ frames, uint32_t n_frames, const uint32_t *__restrict__ narrow_flags, uint32_t *__restrict__ list) {
    if (threadIdx.x == 0) list[0] = 0;
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n_frames; i += blockDim.x)
        if (narrow_flags[frames[i].status_idx]) list[1 + atomicAdd(list, 1u)] = i;
}

// ---- the chroma window of reconstruct420_kernel -------------------------------------------------------------------------
// A CTA of reconstruct420_kernel covers 32 luma block columns x kRows420 luma block rows, one warp per row (kRows420 = 4 is
// b2's CTA). Its chroma window holds, per component, the kRows420 / 2 chroma block rows under the tile plus the line above and
// the line below (kLines lines) and, per line, the 128 columns under the tile plus the column either side. Line l is chroma
// line 4 kRows420 blockIdx.y - 1 + l, column i is chroma column 128 blockIdx.x - 4 + i: a lane's own four samples start at
// i = 4 + 4 lane (an aligned 8- / 16-byte load), its left / right neighbour is i = 3 + 4 lane / 8 + 4 lane. (kRows420: internal.hpp,
// which the planner shares. A cropped frame's CTA runs tile blockIdx + (tx0, ty0) in place of blockIdx: the same window.)
constexpr int kThreads420 = 32 * kRows420;
static_assert(kRows420 % 2 == 0 && kRows420 >= 4 && kRows420 <= 8, "whole chroma block rows, enough warps for phase 1, at most 8 warps");

// The luma tile `ys` in front of the window holds a sample per (coefficient, thread): int16 in the int16 instance for the packed
// and the planar 8-bit stores (Tile420), which then run six CTAs per SM (kWarps420); int32 in the int32 instance (the exact
// path) and for the other kinds, which stay at five.
template <typename T, typename Y = int>
struct Window420 {
    static constexpr int kLines = 4 * kRows420 + 2;
    static constexpr int kLineBytes = 136 * (int)sizeof(T);  // [3 unused][left][128][right][3 unused]
    // + 4 samples: Cr lies two banks off Cb for the int16 stores of phase 1, and 16-byte aligned for the int32 loads
    static constexpr int kCompBytes = kLines * kLineBytes + 4 * (int)sizeof(T);
    static constexpr int kYsBytes = 64 * kThreads420 * (int)sizeof(Y);  // the luma tile `ys` in front of the window
    static constexpr int kSmemBytes = kYsBytes + 2 * kCompBytes;
};
template <typename T, int K>
using Tile420 = std::conditional_t<sizeof(T) == 2 && (K == kStoreCanvas || K == kStorePlanar), int16_t, int>;

__device__ __forceinline__ uint32_t lds32(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint2 lds64(uint32_t a) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint4 lds128(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ int lds_s16(uint32_t a) {
    int v;
    asm volatile("ld.shared.s16 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts16(uint32_t a, int v) { asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "h"((short)v) : "memory"); }
__device__ __forceinline__ void sts32(uint32_t a, int v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }

// x, which the compiler cannot see through: what is derived from it is computed where it is used
__device__ __forceinline__ int opaque(int x) {
    asm volatile("mov.b32 %0, %0;" : "+r"(x));
    return x;
}

// one window sample (T = short / int) at a shared-space byte address
template <typename T>
__device__ __forceinline__ int win_load(uint32_t a) {
    return sizeof(T) == 2 ? lds_s16(a) : (int)lds32(a);
}
template <typename T>
__device__ __forceinline__ void win_store(uint32_t a, int v) {
    if (sizeof(T) == 2) sts16(a, v);
    else sts32(a, v);
}
// two horizontally adjacent window samples, the first at an even column: one 32- / 64-bit store
template <typename T>
__device__ __forceinline__ void win_store2(uint32_t a, int v0, int v1) {
    if (sizeof(T) == 2) sts32(a, (int)(((uint32_t)v0 & 0xffffu) | ((uint32_t)v1 << 16)));
    else asm volatile("st.shared.v2.u32 [%0], {%1,%2};" ::"r"(a), "r"(v0), "r"(v1) : "memory");
}

// ---- b2 ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// NW samples of line y of a sample plane starting at column x0. Away from the frame edge this is a plain run;
// at the edge the clamped addressing reproduces dest[-1] = dest[0], dest[width] = dest[width-1]
// (upsamplerbase.cpp:322-323) and the duplicated first / last line (upsampler.cpp:100-106).
template <int NW, typename T>
__device__ __forceinline__ void load_row(const T *__restrict__ plane, uint32_t pitch, int y, int x0, int cw, int ch, bool interior, int (&v)[NW]) {
    if (interior) {
        const T *row = plane + (uint64_t)y * pitch + x0;
#pragma unroll
        for (int j = 0; j < NW; j++) v[j] = __ldg(row + j);
    } else {
        const T *row = plane + (uint64_t)clampi(y, 0, ch - 1) * pitch;
#pragma unroll
        for (int j = 0; j < NW; j++) v[j] = __ldg(row + clampi(x0 + j, 0, cw - 1));
    }
}

// The same window for a warp whose 32 blocks all lie inside the plane horizontally: a lane fetches its own 8/SX samples
// with 16-byte loads (4 instead of 24 L1 wavefronts per warp instruction) and, for SX == 2, the two neighbouring columns
// xl, xr (already clamped = the edge replication above) with one load each; the line is clamped here.
template <int NW, int SX, typename T>
__device__ __forceinline__ void load_row_own(const T *__restrict__ plane, uint32_t pitch, int y, int ch, uint32_t bx, int xl, int xr, int (&v)[NW]) {
    const T *row = plane + (uint64_t)clampi(y, 0, ch - 1) * pitch;
    if (sizeof(T) == 2) {
        if (SX == 2) {
            const uint2 a = __ldg(reinterpret_cast<const uint2 *>(row) + bx);
            v[0] = __ldg(row + xl), v[NW - 1] = __ldg(row + xr);
            v[1] = (int)(short)(a.x & 0xffffu), v[2] = (int)a.x >> 16, v[3] = (int)(short)(a.y & 0xffffu), v[4] = (int)a.y >> 16;
        } else {
            const uint4 a = __ldg(reinterpret_cast<const uint4 *>(row) + bx);
            v[0] = (int)(short)(a.x & 0xffffu), v[1] = (int)a.x >> 16, v[2] = (int)(short)(a.y & 0xffffu), v[3] = (int)a.y >> 16;
            v[NW - 4] = (int)(short)(a.z & 0xffffu), v[NW - 3] = (int)a.z >> 16, v[NW - 2] = (int)(short)(a.w & 0xffffu), v[NW - 1] = (int)a.w >> 16;
        }
    } else if (SX == 2) {
        const int4 a = __ldg(reinterpret_cast<const int4 *>(row) + bx);
        v[0] = __ldg(row + xl), v[1] = a.x, v[2] = a.y, v[3] = a.z, v[4] = a.w, v[NW - 1] = __ldg(row + xr);
    } else {
        const int4 a = __ldg(reinterpret_cast<const int4 *>(row) + 2 * bx), b = __ldg(reinterpret_cast<const int4 *>(row) + 2 * bx + 1);
        v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w, v[NW - 4] = b.x, v[NW - 3] = b.y, v[NW - 2] = b.z, v[NW - 1] = b.w;
    }
}

// HorizontalFilterCore<2> on a window w[0..5] (w[j] = sample at subsampled x0 - 1 + j): upsampler.cpp:283-307.
__device__ __forceinline__ void hfilter2(const int (&w)[6], int (&o)[8]) {
    o[7] = WADD(WADD(w[5], WMUL(3, w[4])), 1) >> 2;
    o[6] = WADD(WADD(w[3], WMUL(3, w[4])), 2) >> 2;
    o[5] = WADD(WADD(w[4], WMUL(3, w[3])), 1) >> 2;
    o[4] = WADD(WADD(w[2], WMUL(3, w[3])), 2) >> 2;
    o[3] = WADD(WADD(w[3], WMUL(3, w[2])), 1) >> 2;
    o[2] = WADD(WADD(w[1], WMUL(3, w[2])), 2) >> 2;
    o[1] = WADD(WADD(o[2], WMUL(3, w[1])), 1) >> 2;  // reads the freshly written out[2] (upsampler.cpp:301-302)
    o[0] = WADD(WADD(w[0], WMUL(3, w[1])), 2) >> 2;
}

__device__ __forceinline__ int sat_u8_64(long long v) { return (int)(v < 0 ? 0 : (v > 255 ? 255 : v)); }
// four values -> four bytes, each saturated to 0..255 (CLAMP(255, v)), p0 in the low byte: two I2IP instead of four
// conversions plus the shifts and ORs
__device__ __forceinline__ uint32_t pack_sat4(int p0, int p1, int p2, int p3) {
    uint32_t hi, w;
    asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(hi) : "r"(p3), "r"(p2), "r"(0));
    asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(w) : "r"(p1), "r"(p0), "r"(hi));
    return w;
}

// ---- destinations (StoreKind): the canvas kind stores into the batch's output buffer, the described kinds read the
// frame's four b200jpg_plane descriptors at 4 * status_idx of the table b200jpg_batch_decode_into uploads; the float kinds
// carry the conversion map next to the table pointer, as a launch argument
template <int K>
using StoreDst = std::conditional_t<K == kStoreCanvas, uint8_t *, std::conditional_t<kFloatKind<K>, FloatDst, const b200jpg_plane *>>;

__device__ __forceinline__ const b200jpg_plane *planes_of(const b200jpg_plane *p) { return p; }
__device__ __forceinline__ const b200jpg_plane *planes_of(const FloatDst &d) { return d.planes; }

// ---- float elements: convert_bits / map_int / table_at / pick4 / store_elem (store_sm90.cuh)
// byte k of a packed word of four 8-bit samples as 0x4B0000vv: bytes 4..7 of the permute are those of 0x4B000000; with the
// sample tables t, the byte alone (bytes 4..7 of the permute are zero) indexes component c's table
__device__ __forceinline__ float convert_byte(uint32_t w, int k, const float *t, uint32_t c, float s, float b) {
    if (t) return table_at(t, c, __byte_perm(w, 0u, 0x4440u | (uint32_t)k));
    return convert_bits(__byte_perm(w, 0x4B000000u, 0x7440u | (uint32_t)k), s, b);
}
__device__ __forceinline__ uint32_t pack2(int type, float lo, float hi) {
    if (type == B200JPG_SAMPLE_F16) {
        const __half2 h = __floats2half2_rn(lo, hi);
        return *reinterpret_cast<const uint32_t *>(&h);
    }
    const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const uint32_t *>(&h);
}
// the first xmax + 1 of eight converted samples from o on: a whole 16-byte aligned planar row leaves as one 16-byte store
// (fp16 / bf16) or two (fp32), else one store per element
template <int K>
__device__ __forceinline__ void store_row_f(int type, const b200jpg_plane *p, uint8_t *o, const float (&y)[8], int xmax) {
    const bool f32 = type == B200JPG_SAMPLE_F32;
    if (kBaseKind<K> == kStorePlanarF && xmax == 7 && (reinterpret_cast<uintptr_t>(o) & 15u) == 0) {
        uint4 *o4 = reinterpret_cast<uint4 *>(o);
        if (f32) {
            o4[0] = make_uint4(__float_as_uint(y[0]), __float_as_uint(y[1]), __float_as_uint(y[2]), __float_as_uint(y[3]));
            o4[1] = make_uint4(__float_as_uint(y[4]), __float_as_uint(y[5]), __float_as_uint(y[6]), __float_as_uint(y[7]));
        } else {
            o4[0] = make_uint4(pack2(type, y[0], y[1]), pack2(type, y[2], y[3]), pack2(type, y[4], y[5]), pack2(type, y[6], y[7]));
        }
        return;
    }
    const int64_t s = (kBaseKind<K> == kStorePlanarF) ? (f32 ? 4 : 2) : p->bytes_per_pixel;
#pragma unroll
    for (int x = 0; x < 8; x++)
        if (x <= xmax) store_elem(type, o + x * s, y[x]);
}

// the sample (x, y) of a described component: plane_at (store_sm90.cuh)

// the first xmax + 1 of eight 8-bit samples (w0 | w1, sample 0 in the low byte of w0) from o on: one 8-byte store for a whole
// aligned planar row, else one store per sample
template <int K>
__device__ __forceinline__ void store_row8(const b200jpg_plane *p, uint8_t *o, uint32_t w0, uint32_t w1, int xmax) {
    if (K == kStorePlanar && xmax == 7 && (reinterpret_cast<uintptr_t>(o) & 7u) == 0) {
        *reinterpret_cast<uint2 *>(o) = make_uint2(w0, w1);
        return;
    }
    const int64_t s = (K == kStorePlanar) ? 1 : p->bytes_per_pixel;
#pragma unroll
    for (int x = 0; x < 8; x++)
        if (x <= xmax) o[x * s] = (uint8_t)(((x < 4) ? w0 : w1) >> (8 * (x & 3)));
}

// one block row of component c of a described destination, the eight clamped samples packed in w0 | w1: as bytes, or
// converted for the float kinds
template <int K, typename D>
__device__ __forceinline__ void store_row(const D &out, int c, const b200jpg_plane *p, uint8_t *o, uint32_t w0, uint32_t w1, int xmax) {
    if constexpr (kFloatKind<K>) {
        float y[8];
#pragma unroll
        for (int x = 0; x < 8; x++) y[x] = convert_byte((x < 4) ? w0 : w1, x & 3, table_of<kTableKind<K>>(out), (uint32_t)c, out.scale[c], out.bias[c]);
        store_row_f<K>(out.type, p, o, y, xmax);
    } else {
        store_row8<K>(p, o, w0, w1, xmax);
    }
}

// ---- kStoreRuns / kStoreRunsF: the lane's block has been staged in its luma tile column -- line y of component c in the words
// st[(8 y + 2 c) NT] and st[(8 y + 2 c + 1) NT], eight clamped 8-bit samples, sample 0 in the low byte -- and leaves here. Exif
// orientations make the rewritten descriptors of a [N, C, H, W] tensor or of the packed slot contiguous along x in descending
// order (mirrored rows) or along y in either order (transposed): such runs of eight samples leave as one vector store each.
__device__ __forceinline__ uint32_t byte_of(uint32_t w, int k) { return (w >> (8 * k)) & 0xffu; }
__device__ __forceinline__ uint32_t rev4(uint32_t w) { return __byte_perm(w, 0u, 0x0123u); }

// eight samples in memory order (w0 | w1) at o, stride e: one 8-byte store when aligned
__device__ __forceinline__ void put_run8(uint8_t *o, uint32_t w0, uint32_t w1) {
    if ((reinterpret_cast<uintptr_t>(o) & 7u) == 0) {
        *reinterpret_cast<uint2 *>(o) = make_uint2(w0, w1);
        return;
    }
#pragma unroll
    for (int k = 0; k < 8; k++) o[k] = (uint8_t)byte_of(k < 4 ? w0 : w1, k & 3);
}
// the same converted to float elements of `type`: 16-byte stores when aligned
__device__ __forceinline__ void put_run_f(int type, uint8_t *o, uint32_t w0, uint32_t w1, const float *t, uint32_t c, float s, float b) {
    float y[8];
#pragma unroll
    for (int k = 0; k < 8; k++) y[k] = convert_byte(k < 4 ? w0 : w1, k & 3, t, c, s, b);
    const bool f32 = type == B200JPG_SAMPLE_F32;
    if ((reinterpret_cast<uintptr_t>(o) & 15u) == 0) {
        uint4 *o4 = reinterpret_cast<uint4 *>(o);
        if (f32) {
            o4[0] = make_uint4(__float_as_uint(y[0]), __float_as_uint(y[1]), __float_as_uint(y[2]), __float_as_uint(y[3]));
            o4[1] = make_uint4(__float_as_uint(y[4]), __float_as_uint(y[5]), __float_as_uint(y[6]), __float_as_uint(y[7]));
        } else {
            o4[0] = make_uint4(pack2(type, y[0], y[1]), pack2(type, y[2], y[3]), pack2(type, y[4], y[5]), pack2(type, y[6], y[7]));
        }
        return;
    }
    const int e = f32 ? 4 : 2;
#pragma unroll
    for (int k = 0; k < 8; k++) store_elem(type, o + k * e, y[k]);
}

template <int K, typename D>
__device__ __forceinline__ void put_run(const D &out, int c, uint8_t *o, uint32_t w0, uint32_t w1) {
    if constexpr (kBaseKind<K> == kStoreRunsF) put_run_f(out.type, o, w0, w1, table_of<kTableKind<K>>(out), (uint32_t)c, pick4(out.scale, c), pick4(out.bias, c));
    else put_run8(o, w0, w1);
}

struct PlaneDesc {
    uint64_t data;
    int64_t bpp, bpr;
};
__device__ __forceinline__ PlaneDesc desc_of(const b200jpg_plane *p) {
    PlaneDesc d;
    int bpp;
    asm volatile("ld.global.nc.u64 %0, [%1];" : "=l"(d.data) : "l"(&p->data));
    asm volatile("ld.global.nc.s32 %0, [%1];" : "=r"(bpp) : "l"(&p->bytes_per_pixel));
    asm volatile("ld.global.nc.u64 %0, [%1];" : "=l"(d.bpr) : "l"(&p->bytes_per_row));
    d.bpp = bpp;
    return d;
}

// column x (0..7) of component c, rows 0..3 and 4..7 of the staged block, row 0 in the low byte
template <uint32_t NT>
__device__ __forceinline__ void staged_column(const int *st, int c, int x, uint32_t &lo, uint32_t &hi) {
    uint32_t w[8];
#pragma unroll
    for (int y = 0; y < 8; y++) w[y] = (uint32_t)st[(8 * y + 2 * c + (x >> 2)) * NT];
    const uint32_t k = (uint32_t)(x & 3), sel = k | ((4u + k) << 4);  // bytes k of two words -> bytes 0, 1
    lo = __byte_perm(__byte_perm(w[0], w[1], sel), __byte_perm(w[2], w[3], sel), 0x5410u);
    hi = __byte_perm(__byte_perm(w[4], w[5], sel), __byte_perm(w[6], w[7], sel), 0x5410u);
}

// The store phase of kStoreRuns / kStoreRunsF for the valid lane's block at (X, Y), samples xmin <= x <= xmax, ymin <= y <= ymax
// (xmin = ymin = 0 unless kClipKind<K>: a block cut by the crop's left or top edge). A run of eight leaves whole or not at all.
template <int K, int NC, uint32_t NT, typename D>
__device__ __forceinline__ void store_staged(const D &out, const b200jpg_plane *pl, const int *st, int X, int Y, int xmin, int xmax, int ymin, int ymax) {
    constexpr int KB = kBaseKind<K>;
    if constexpr (!kClipKind<K>) xmin = ymin = 0;
    int64_t e = 1;  // element size
    if constexpr (KB == kStoreRunsF) e = out.type == B200JPG_SAMPLE_F32 ? 4 : 2;
    if constexpr (KB == kStoreRuns && NC == 3) {
        // the packed slot seen as an interleaved bitmap: three components one byte apart with one pair of strides
        const PlaneDesc d0 = desc_of(pl), d1 = desc_of(pl + 1), d2 = desc_of(pl + 2);
        const bool inter = d1.data == d0.data + 1 && d2.data == d0.data + 2 && d1.bpp == d0.bpp && d2.bpp == d0.bpp && d1.bpr == d0.bpr &&
                           d2.bpr == d0.bpr;
        const bool along_x = inter && (d0.bpp == 3 || d0.bpp == -3) && xmin == 0 && xmax == 7,
                   along_y = inter && (d0.bpr == 3 || d0.bpr == -3) && ymin == 0 && ymax == 7;
        if (along_x || along_y) {
            // run j: line y = j (along x) or column x = j (along y); 24 bytes of eight pixels in memory order from the lowest one
            const int64_t step = along_x ? d0.bpp : d0.bpr;
            const int jmin = along_x ? ymin : xmin, jmax = along_x ? ymax : xmax;
#pragma unroll 1
            for (int j = jmin; j <= jmax; j++) {
                uint32_t cl[3], ch[3];  // component c's eight samples of the run, in run order (k = 0 first)
#pragma unroll
                for (int c = 0; c < 3; c++) {
                    if (along_x) cl[c] = (uint32_t)st[(8 * j + 2 * c) * NT], ch[c] = (uint32_t)st[(8 * j + 2 * c + 1) * NT];
                    else staged_column<NT>(st, c, j, cl[c], ch[c]);
                    if (step < 0) {
                        const uint32_t t = rev4(cl[c]);
                        cl[c] = rev4(ch[c]);
                        ch[c] = t;
                    }
                }
                uint32_t wd[6];
#pragma unroll
                for (int q = 0; q < 6; q++) {
                    uint32_t v = 0;
#pragma unroll
                    for (int b = 0; b < 4; b++) {
                        const int i = 4 * q + b, p = i / 3, c = i % 3;
                        v |= byte_of(p < 4 ? cl[c] : ch[c], p & 3) << (8 * b);
                    }
                    wd[q] = v;
                }
                const int x = along_x ? (step < 0 ? 7 : 0) : j, y = along_x ? j : (step < 0 ? 7 : 0);
                uint8_t *o = reinterpret_cast<uint8_t *>(d0.data + (uint64_t)((int64_t)(X + x) * d0.bpp) + (uint64_t)((int64_t)(Y + y) * d0.bpr));
                if ((reinterpret_cast<uintptr_t>(o) & 7u) == 0) {
                    uint2 *o2 = reinterpret_cast<uint2 *>(o);
#pragma unroll
                    for (int q = 0; q < 3; q++) o2[q] = make_uint2(wd[2 * q], wd[2 * q + 1]);
                } else if ((reinterpret_cast<uintptr_t>(o) & 3u) == 0) {
#pragma unroll
                    for (int q = 0; q < 6; q++) reinterpret_cast<uint32_t *>(o)[q] = wd[q];
                } else {
#pragma unroll
                    for (int i = 0; i < 24; i++) o[i] = (uint8_t)byte_of(wd[i >> 2], i & 3);
                }
            }
            return;
        }
    }
#pragma unroll 1
    for (int c = 0; c < NC; c++) {
        const PlaneDesc d = desc_of(pl + c);
        auto at = [&](int x, int y) { return reinterpret_cast<uint8_t *>(d.data + (uint64_t)((int64_t)(X + x) * d.bpp) + (uint64_t)((int64_t)(Y + y) * d.bpr)); };
        if ((d.bpp == e || d.bpp == -e) && xmin == 0 && xmax == 7) {  // rows are runs (mirrored: descending)
#pragma unroll 1
            for (int y = ymin; y <= ymax; y++) {
                const uint32_t w0 = (uint32_t)st[(8 * y + 2 * c) * NT], w1 = (uint32_t)st[(8 * y + 2 * c + 1) * NT];
                if (d.bpp > 0) put_run<K>(out, c, at(0, y), w0, w1);
                else put_run<K>(out, c, at(7, y), rev4(w1), rev4(w0));
            }
        } else if ((d.bpr == e || d.bpr == -e) && ymin == 0 && ymax == 7) {  // columns are runs (transposed)
#pragma unroll 1
            for (int x = xmin; x <= xmax; x++) {
                uint32_t lo, hi;
                staged_column<NT>(st, c, x, lo, hi);
                if (d.bpr > 0) put_run<K>(out, c, at(x, 0), lo, hi);
                else put_run<K>(out, c, at(x, 7), rev4(hi), rev4(lo));
            }
        } else {  // partial blocks at the frame (or crop) edge, or a layout without a contiguous axis: one store per sample
#pragma unroll 1
            for (int y = ymin; y <= ymax; y++)
#pragma unroll 1
                for (int x = xmin; x <= xmax; x++) {
                    const uint32_t v = byte_of((uint32_t)st[(8 * y + 2 * c + (x >> 2)) * NT], x & 3);
                    if constexpr (KB == kStoreRunsF) store_elem(out.type, at(x, y), map_int(table_of<kTableKind<K>>(out), c, (int)v, pick4(out.scale, c), pick4(out.bias, c)));
                    else *at(x, y) = (uint8_t)v;
                }
        }
    }
}

// ycbcrtrafo.cpp:842-850 with the matrix of colortransformerfactory.cpp:136-138 (13 fractional bits) and
// FIX_COLOR_TO_INT (tools/numerics.hpp:65).  The reference multiplies in 64 bits; 32 bits give the same result
// while |y|, |cb|, |cr| <= 65535 -- blocks that violate that (damaged streams only) are flagged `wide`.
// The results are NOT yet clamped (pack_sat4 does that), except in the 64-bit mode.
template <int MODE>  // 0: 32-bit YCbCr, 1: 64-bit YCbCr (samples outside the guarded range), 2: identity
__device__ __forceinline__ void to_rgb(int y, int cbv, int crv, int &r, int &g, int &b) {
    if (MODE == 2) {  // COLOR_TO_INT (tools/numerics.hpp:69)
        r = WADD(y, 8) >> 4;
        g = WADD(cbv, 8) >> 4;
        b = WADD(crv, 8) >> 4;
        return;
    }
    const int cb = WSUB(cbv, 128 << 4), cr = WSUB(crv, 128 << 4);
    if (MODE == 0) {
        const int yy = y * 8192 + 65536;
        r = (yy + cr * 11485) >> 17;
        g = (yy - cb * 2819 - cr * 5850) >> 17;
        b = (yy + cb * 14516) >> 17;
    } else {
        const long long Y = y, CB = cb, CR = cr;
        r = sat_u8_64((Y * 8192 + CR * 11485 + 65536) >> 17);
        g = sat_u8_64((Y * 8192 - CB * 2819 - CR * 5850 + 65536) >> 17);
        b = sat_u8_64((Y * 8192 + CB * 14516 + 65536) >> 17);
    }
}

// ---- the 16-bit tile of reconstruct420_kernel<int16_t> (Tile420) ----------------------------------------------------------
// Warp w owns the 4 KB from byte 4096 w on, laid out [coefficient][lane]: sample (c, lane) at 2 (32 c + lane). Its 32 blocks of
// coefficients are exactly those 4 KB, so each block row is reconstructed in place: coefficient row r of the 32 blocks (16-byte
// piece (block b, row r) at 512 r + 16 (b ^ r)) and, once read, the eight row-pass outputs of every lane (at 512 r + 64 k +
// 2 lane) take the same 512 bytes. Banks: 512 r is a multiple of 128, so a piece lands in 16-byte bank group (b ^ r) & 7. A
// 16-byte access is served a quarter warp (eight lanes) at a time: the stores of tile_fetch's piece i * 32 + lane have b = 4 i +
// lane / 8 fixed and r = lane & 7, the per-lane reads b = lane and r fixed, so the eight lanes hit eight different groups
// either way; the int16 samples of a warp are 64 contiguous bytes. All conflict-free. (The int32 tile keeps the pieces in its
// upper half, at the same offsets + 4096: kStash.)
//
// Range. The row pass idct8t<16, 5> of int16 coefficients is out_n = (sum_k W[n][k] v_k + 16) >> 5 with sum_k |W[n][k]| = 3825
// for every n; the negative weights of an output sum to at most 2434 in magnitude (n = 1), the positive ones to 3825 (n = 0). So
// over v in [-32768, 32767]^8 the outputs lie in [(-(32767 * 3825 + 3825) + 16) >> 5, (32767 * 3825 + 2434 + 16) >> 5] =
// [-3,916,800, 3,916,757], 120 times the int16 range (tests/test_recon420_tile16_cpu.py): a stored output can wrap. Every
// output goes through the min / max of its lane before it is stored, and a warp with one outside int16 flags the frame `narrow`
// (the int32 instance redoes it) -- the min / max the column pass kept for the 32-bit colour range moves here: with the row
// outputs inside int16 the column pass gives |out| <= (3825 * 32768 + 2048) >> 12 = 30,600, nothing is `wide`.
// The level shift is left out of the row pass: dcoffset << 3 = 1024 on the DC adds exactly 512 * 1024 = 16384 << 5 to every
// output of coefficient row 0, and that row's outputs add exactly 512 * 16384 = 2048 << 12 to every column-pass output. So the
// row pass runs without it and the column pass rounds with 2048 + (2048 << 12) (kRound16): the same sums, bit for bit, with
// the tile centred on zero -- row 0 of a flat block of 255 is 16256 instead of 32640, and real images stay far inside int16.
constexpr int kRound16 = 2048 + (2048 << 12);

// the 16-byte pieces of a warp's 32 blocks, eight per lane (piece i * 32 + lane: block 4 i + lane / 8, row lane & 7), into the
// warp's tile at byte offset kStash (0 for the int16 tile, 4096 for the upper half of the int32 one)
template <uint32_t kStash>
__device__ __forceinline__ void tile_stash_at(uint32_t wseg, const uint4 (&pc)[8]) {
    const uint32_t lane = threadIdx.x & 31, prow = lane & 7u, sub = lane >> 3;
#pragma unroll
    for (uint32_t i = 0; i < 8; i++) {
        const uint32_t blk = 4u * i + sub;
        const uint32_t dst = wseg + kStash + 512u * prow + 128u * (blk >> 3) + 16u * ((blk & 7u) ^ prow);
        asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(dst), "r"(pc[i].x), "r"(pc[i].y), "r"(pc[i].z), "r"(pc[i].w) : "memory");
    }
    __syncwarp();
}

// The row pass of the int16 tile yw (the warp's 4 KB) in place, coefficient rows 0 .. kRows - 1, without the level shift
// (kRound16); mn / mx: the min / max of the outputs (both start at 0)
template <int kRows>
__device__ __forceinline__ void tile_rows16(int16_t *yw, int &mn, int &mx) {
    const uint32_t lane = threadIdx.x & 31;
    int16_t *my = yw + lane;
    const uint32_t wseg = (uint32_t)__cvta_generic_to_shared(yw);
    auto piece = [&](int r) { return lds128(wseg + 512u * (uint32_t)r + 16u * (lane ^ (uint32_t)r)); };
    mn = 0, mx = 0;
    uint4 q = piece(0);
#pragma unroll 1
    for (int r = 0; r < kRows; r++) {
        const uint4 qn = piece((r < kRows - 1) ? r + 1 : r);
        int v[8];
        unpack_row_raw(q, v);
        idct8t<16, 5>(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
        mx = __vimax3_s32(__vimax3_s32(mx, v[0], v[1]), __vimax3_s32(v[2], v[3], v[4]), __vimax3_s32(v[5], v[6], v[7]));
        mn = __vimin3_s32(__vimin3_s32(mn, v[0], v[1]), __vimin3_s32(v[2], v[3], v[4]), __vimin3_s32(v[5], v[6], v[7]));
        __syncwarp();  // every lane has read piece r before it is overwritten
#pragma unroll
        for (int k = 0; k < 8; k++) my[(8 * r + k) * 32] = (int16_t)v[k];
        q = qn;
    }
}

// kWin: the chroma samples come from the window of reconstruct420_kernel at shared-space address `win` instead of the sample
// planes. chroma_wide: a chroma sample the tile reads may leave the 32-bit colour range.
// K: the destination kind (StoreKind). KS > 1: the frame is downscaled by KS (B200JPG_FLAG_DOWNSCALE_k) -- the luma of an output
// block comes from the KS x KS coefficient blocks under it through scaled_idct_block instead of the 8x8 IDCT of one block.
// NO = 3 with NC = 1 (B200JPG_FLAG_OUTPUT_RGB, described kinds only): the grey row leaves through the descriptors of components 0, 1
// and 2, each converted with its own component's map.
// YT = int16_t (reconstruct420_kernel<int16_t>, Canvas and Planar): the luma tile is the warp's 4 KB of the 16-bit tile
// (tile_rows16), and a row-pass output outside int16 flags the frame in `narrow`.
template <int NC, int SX, int SY, typename T, bool kWin = false, int K = kStoreCanvas, int KS = 1, int NO = NC, typename YT = int>
__device__ __forceinline__ void reconstruct_tile(const FrameRecon &f, YT *ys, const int16_t *__restrict__ coef, const T *__restrict__ samples,
                                                 uint32_t win, bool chroma_wide, StoreDst<K> __restrict__ out, uint32_t *__restrict__ narrow = nullptr) {
    static_assert(!kWin || (NC == 3 && SX == 2 && SY == 2), "the chroma window is 4:2:0 only");
    constexpr bool k16 = sizeof(YT) == 2;
    static_assert(!k16 || (kWin && KS == 1 && sizeof(T) == 2 && std::is_same<YT, Tile420<T, K>>::value), "the 16-bit tile is reconstruct420_kernel<int16_t>'s");
    constexpr uint32_t NT = kWin ? kThreads420 : kThreadsB;  // threads per CTA: the stride of the tile [coefficient][thread]
    constexpr uint32_t TS = k16 ? 32u : NT;                  // the stride of a lane's samples in its tile
    constexpr int KB = kBaseKind<K>;
    constexpr bool kClip = kClipKind<K>;  // a cropped frame: tile (tx0, ty0) + blockIdx, stores inside the clip rectangle only
    constexpr bool kRep = NC == 1 && NO == 3;
    static_assert(NO == NC || (kRep && KB != kStoreCanvas), "a grey frame leaves as three components through descriptors only");
    const uint32_t W = f.width, H = f.height;
    // blocks that carry visible pixels (cropped: pixels inside the clip rectangle)
    const uint32_t vbw = ((kClip ? f.clip_x1 : W) + 7) >> 3, vbh = ((kClip ? f.clip_y1 : H) + 7) >> 3;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t tile_x = kClip ? f.tx0 + blockIdx.x : blockIdx.x, tile_y = kClip ? f.ty0 + blockIdx.y : blockIdx.y;
    const uint32_t bx0 = tile_x * 32, bx = bx0 + lane, by = tile_y * (NT / 32) + warp;
    if (by >= vbh) return;  // whole warp
    if (kClip && by < (f.clip_y0 >> 3)) return;
    const bool valid = bx < vbw && (!kClip || bx >= (f.clip_x0 >> 3));
    const int X = 8 * (int)bx, Y = 8 * (int)by;
    YT *my = k16 ? ys + 2048u * warp + lane : ys + threadIdx.x;

    int mx = 0, mn = 0;
    if constexpr (k16) {
        // ---- luma coefficients: 4 KB of contiguous HBM for the warp's 32 blocks, eight coalesced 16-byte loads per lane, then
        // the row pass in place (tile_rows16) and its range check
        const uint4 *src = reinterpret_cast<const uint4 *>(coef + f.coef_base[0] + ((uint64_t)by * f.bw[0] + bx0) * 64u);
        const uint32_t sub = lane >> 3;
        uint4 pc[8];
#pragma unroll
        for (uint32_t i = 0; i < 8; i++) pc[i] = (bx0 + 4u * i + sub < f.bw[0]) ? __ldg(src + i * 32u + lane) : make_uint4(0u, 0u, 0u, 0u);
        YT *yw = ys + 2048u * warp;
        tile_stash_at<0>((uint32_t)__cvta_generic_to_shared(yw), pc);
        tile_rows16<8>(yw, mn, mx);
        if (mx > 32767 || mn < -32768) atomicOr(narrow + f.status_idx, 1u);  // `narrow`: the int32 instance redoes the frame
        // ---- column pass (:291-334), the level shift in the rounding (kRound16)
#pragma unroll 1
        for (int k = 0; k < 8; k++) {
            int v[8];
#pragma unroll
            for (int r = 0; r < 8; r++) v[r] = my[(8 * r + k) * 32];
            idct8t<kRound16, 12>(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
#pragma unroll
            for (int r = 0; r < 8; r++) my[(8 * r + k) * 32] = (int16_t)v[r];
        }
        mx = mn = 0;  // |luma| <= 30,600 + 2048: never `wide`
    } else if constexpr (KS > 1) {
        // ---- downscaled: output block (bx, by) holds the (8/KS) x (8/KS) samples of coefficient blocks (KS bx + i, KS by + j)
        constexpr int N = 8 / KS;
#pragma unroll 1
        for (int j = 0; j < KS; j++) {
#pragma unroll 1
            for (int i = 0; i < KS; i++) {
                const uint32_t cx = KS * bx + i, cy = KS * by + j;
                int sm[N][N];
                if (cx < f.coef_bw[0] && cy < f.coef_bh[0]) {
                    scaled_idct_block<KS>(coef + f.coef_base[0] + ((uint64_t)cy * f.coef_bw[0] + cx) * 64u, 128 << 4, sm);
                } else {
#pragma unroll
                    for (int n = 0; n < N; n++)
#pragma unroll
                        for (int m = 0; m < N; m++) sm[n][m] = 0;  // beyond the coefficient grid: never visible
                }
#pragma unroll
                for (int n = 0; n < N; n++)
#pragma unroll
                    for (int m = 0; m < N; m++) {
                        my[(8 * (N * j + n) + N * i + m) * NT] = sm[n][m];
                        mx = max(mx, sm[n][m]);
                        mn = min(mn, sm[n][m]);
                    }
            }
        }
    } else {
        // ---- luma coefficients: the warp's 32 blocks are 4 KB of contiguous HBM. Eight coalesced 16-byte loads per lane
        // (four full lines per warp instruction instead of 32 partial ones) park them in the upper half of the warp's tile
        // columns, 16-byte piece (block, row) at row segment 32 + 4*row + block/8, slot (block%8) ^ row: conflict-free for
        // these writes and for the per-lane reads below. The row pass overwrites a segment only after its piece was consumed.
        {
            const uint32_t wseg = (uint32_t)__cvta_generic_to_shared(ys) + 128u * warp;  // bytes; row segment j at + 4*NT*j
            const uint4 *src = reinterpret_cast<const uint4 *>(coef + f.coef_base[0] + ((uint64_t)by * f.bw[0] + bx0) * 64u);
            const uint32_t prow = lane & 7u, sub = lane >> 3;
            uint4 pc[8];
    #pragma unroll
            for (uint32_t i = 0; i < 8; i++) {
                const bool have = bx0 + 4u * i + sub < f.bw[0];  // past the end of the block row: nothing (those lanes store nothing)
                pc[i] = have ? __ldg(src + i * 32u + lane) : make_uint4(0u, 0u, 0u, 0u);
            }
    #pragma unroll
            for (uint32_t i = 0; i < 8; i++) {
                const uint32_t blk = 4u * i + sub;
                const uint32_t dst = wseg + 4u * NT * (32u + 4u * prow + (blk >> 3)) + 16u * ((blk & 7u) ^ prow);
                asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(dst), "r"(pc[i].x), "r"(pc[i].y), "r"(pc[i].z), "r"(pc[i].w) : "memory");
            }
            __syncwarp();
            // ---- row pass (dct/idct.cpp:237-287): the next row's piece is read before this row's results are written
            const uint32_t mine = wseg + 4u * NT * (32u + (lane >> 3));
            auto piece = [&](int r) {
                uint4 q;
                asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
                             : "=r"(q.x), "=r"(q.y), "=r"(q.z), "=r"(q.w)
                             : "r"(mine + 16u * NT * (uint32_t)r + 16u * ((lane & 7u) ^ (uint32_t)r))
                             : "memory");
                return q;
            };
            uint4 q = piece(0);
    #pragma unroll 1
            for (int r = 0; r < 8; r++) {
                const uint4 qn = piece((r < 7) ? r + 1 : r);
                int v[8];
                unpack_row_raw(q, v);
                if (r == 0) v[0] = WADD(v[0], 128 << 3);  // dcoffset << 3 (idct.cpp:233,244), preshift folded into the rounding (unpack_row_raw)
                idct8t<16, 5>(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
                __syncwarp();
    #pragma unroll
                for (int k = 0; k < 8; k++) my[(8 * r + k) * NT] = v[k];
                q = qn;
            }
        }
        // ---- column pass (:291-334) + range guard for the 32-bit colour arithmetic
    #pragma unroll 1
        for (int k = 0; k < 8; k++) {
            int v[8];
    #pragma unroll
            for (int r = 0; r < 8; r++) v[r] = my[(8 * r + k) * NT];
            idct8t<2048, 12>(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
    #pragma unroll
            for (int r = 0; r < 8; r++) my[(8 * r + k) * NT] = v[r];
            mx = __vimax3_s32(__vimax3_s32(mx, v[0], v[1]), v[2], v[3]);
            mx = __vimax3_s32(__vimax3_s32(mx, v[4], v[5]), v[6], v[7]);
            mn = __vimin3_s32(__vimin3_s32(mn, v[0], v[1]), v[2], v[3]);
            mn = __vimin3_s32(__vimin3_s32(mn, v[4], v[5]), v[6], v[7]);
        }
    }

    int xmax = (X + 7 < (int)W) ? 7 : (int)((W - 1) & 7);
    int ymax = (Y + 7 < (int)H) ? 7 : (int)((H - 1) & 7);
    int xmin = 0, ymin = 0;
    if constexpr (kClip) {
        xmin = max((int)f.clip_x0 - X, 0), xmax = min((int)f.clip_x1 - 1 - X, 7);
        ymin = max((int)f.clip_y0 - Y, 0), ymax = min((int)f.clip_y1 - 1 - Y, 7);
    }
    const uint32_t opitch = W * NC;
    uint8_t *obase = nullptr;
    const b200jpg_plane *pl = nullptr;  // described kinds: the frame's component descriptors
    if constexpr (KB == kStoreCanvas) obase = out + f.out_base + (uint64_t)Y * opitch + (uint64_t)X * NC;
    else pl = planes_of(out) + 4u * f.status_idx;

    if (NC == 1) {  // identity, COLOR_TO_INT (numerics.hpp:69) + clamp
        if (!valid) return;
#pragma unroll 1
        for (int r = 0; r <= ymax; r++) {
            uint8_t *o = (KB == kStoreCanvas) ? obase + (uint64_t)r * opitch : ((KB == kStoreRuns || KB == kStoreRunsF) ? nullptr : plane_at(pl, X, Y + r));
            int px[8];
#pragma unroll
            for (int x = 0; x < 8; x++) px[x] = WADD(my[(8 * r + x) * TS], 8) >> 4;
            const uint32_t w0 = pack_sat4(px[0], px[1], px[2], px[3]), w1 = pack_sat4(px[4], px[5], px[6], px[7]);
            if constexpr (KB == kStoreRuns || KB == kStoreRunsF) {  // staged in the line's luma slots, which are consumed
                my[(8 * r) * NT] = (int)w0;
                my[(8 * r + 1) * NT] = (int)w1;
                if constexpr (kRep) {  // the same words as components 1 and 2 of the line
                    my[(8 * r + 2) * NT] = my[(8 * r + 4) * NT] = (int)w0;
                    my[(8 * r + 3) * NT] = my[(8 * r + 5) * NT] = (int)w1;
                }
                continue;
            }
            if (KB == kStoreCanvas) {
                if (xmax == 7 && ((reinterpret_cast<uintptr_t>(o) & 7u) == 0)) {
                    *reinterpret_cast<uint2 *>(o) = make_uint2(w0, w1);
                } else {
#pragma unroll
                    for (int x = 0; x < 8; x++)
                        if (x <= xmax) o[x] = (uint8_t)(((x < 4) ? w0 : w1) >> (8 * (x & 3)));
                }
            } else {
                store_row<K>(out, 0, pl, o, w0, w1, xmax);
                if constexpr (kRep) {
                    store_row<K>(out, 1, pl + 1, plane_at(pl + 1, X, Y + r), w0, w1, xmax);
                    store_row<K>(out, 2, pl + 2, plane_at(pl + 2, X, Y + r), w0, w1, xmax);
                }
            }
        }
        if constexpr (KB == kStoreRuns || KB == kStoreRunsF) store_staged<K, kRep ? 3 : 1, NT>(out, pl, my, X, Y, xmin, xmax, ymin, ymax);
        return;
    }

    constexpr int NW = (SX == 2) ? 6 : 8;
    const int cw = (int)f.cw, ch = (int)f.ch;
    const uint32_t cpitch = 8u * f.bw[1];
    const T *p1 = kWin ? nullptr : samples + f.sample_base[1];
    const T *p2 = kWin ? nullptr : samples + f.sample_base[2];
    const int cx0 = X / SX - ((SX == 2) ? 1 : 0);  // window column 0 (upsampler.cpp:87,108-109)
    const int cy0 = Y / SY;
    const bool ycbcr = f.ycbcr != 0;
    // int16 samples: chroma is inside the guarded range by construction, only this block's luma can leave it
    const bool wide = chroma_wide || mx > kWide || mn < -kWide;
    // the whole window lies inside the plane: no clamping needed
    const bool interior = valid && cx0 >= 0 && cx0 + NW <= cw && cy0 - 1 >= 0 && cy0 + ((SY == 2) ? 5 : 8) <= ch;
    // warp-uniform: every block of the warp is visible and every lane's own samples lie inside the plane
    constexpr int OWN = 8 / SX;
    const bool fast = (bx0 + 32 <= vbw) && ((int)((bx0 + 32) * OWN) <= cw);
    const int xl = (cx0 > 0) ? cx0 : 0, xr = (cx0 + NW - 1 < cw) ? cx0 + NW - 1 : cw - 1;
    const bool lin = cx0 >= 0, rin = cx0 + NW - 1 < cw;  // the window's left / right neighbour columns are not clamped
    // chroma (line 0, column 0) of the shared-memory window (Window420)
    const int wy0 = 4 * (int)(NT / 32) * (int)tile_y - 1, wx0 = 128 * (int)tile_x - 4;
    auto fetch = [&](int y, int (&d1)[NW], int (&d2)[NW]) {
        if (kWin) {
            using Wn = Window420<T>;
            const uint32_t line = win + (uint32_t)(clampi(y, 0, ch - 1) - wy0) * (uint32_t)Wn::kLineBytes;
            constexpr uint32_t S = sizeof(T);
            if (fast) {
#pragma unroll
                for (int c = 0; c < 2; c++) {
                    int (&d)[NW] = c ? d2 : d1;
                    const uint32_t a = line + (uint32_t)c * (uint32_t)Wn::kCompBytes;
                    const uint32_t own = a + (4u + 4u * lane) * S;  // the lane's own four samples
                    if (S == 2) {
                        const uint2 o = lds64(own);
                        d[1] = (int)(short)(o.x & 0xffffu), d[2] = (int)o.x >> 16, d[3] = (int)(short)(o.y & 0xffffu), d[4] = (int)o.y >> 16;
                    } else {
                        const uint4 o = lds128(own);
                        d[1] = (int)o.x, d[2] = (int)o.y, d[3] = (int)o.z, d[4] = (int)o.w;
                    }
                    if constexpr (k16) {
                        // the neighbours are the samples either side of the own four (the halo columns for lanes 0 / 31), unless
                        // the frame edge clamps them onto d[1] / d[4]: immediate offsets, no per-lane columns held in registers
                        d[0] = lin ? win_load<T>(own - S) : d[1];
                        d[NW - 1] = rin ? win_load<T>(own + 4u * S) : d[4];
                    } else {
                        d[0] = win_load<T>(a + (uint32_t)(xl - wx0) * S);
                        d[NW - 1] = win_load<T>(a + (uint32_t)(xr - wx0) * S);
                    }
                }
            } else if (valid) {
                // at the frame edge: the clamped addressing below, always inside the window. 16-bit tile: `opaque` keeps the
                // compiler from hoisting the six columns out of the line loop, where they held registers (and spilled at 80)
                const int c0 = k16 ? opaque(cx0) : cx0;
#pragma unroll
                for (int j = 0; j < NW; j++) {
                    const uint32_t a = line + (uint32_t)(clampi(c0 + j, 0, cw - 1) - wx0) * S;
                    d1[j] = win_load<T>(a);
                    d2[j] = win_load<T>(a + (uint32_t)Wn::kCompBytes);
                }
            }
        } else if (fast) {
            load_row_own<NW, SX, T>(p1, cpitch, y, ch, bx, xl, xr, d1);
            load_row_own<NW, SX, T>(p2, cpitch, y, ch, bx, xl, xr, d2);
        } else if (valid) {
            load_row<NW, T>(p1, cpitch, y, cx0, cw, ch, interior, d1);
            load_row<NW, T>(p2, cpitch, y, cx0, cw, ch, interior, d2);
        }
    };

    // rolling lines: SY == 2 keeps top/cur/bot (upsampler.cpp:92-106), SY == 1 only cur
    int top1[NW], cur1[NW], bot1[NW], top2[NW], cur2[NW], bot2[NW];
    if (SY == 2) {
        fetch(cy0 - 1, top1, top2);
        fetch(cy0 + 1, bot1, bot2);
    }
    fetch(cy0, cur1, cur2);

    auto lines = [&](auto mode_tag) {
        constexpr int MODE = decltype(mode_tag)::value;
        // one output line; for SY == 2 the line parity is a compile-time constant (the loop below is unrolled by two),
        // so the choice of the neighbour line and of the rounding needs no selects
        auto one_line = [&](int r, auto odd_tag) {
            constexpr bool odd = decltype(odd_tag)::value;
            uint32_t wd[6];
            if (valid) {
                int px[24];
                int v1[NW], v2[NW];
                if (SY == 2) {  // VerticalFilterCore<2>, upsampler.cpp:136-168: even lines lean on top, odd lines on bot
                    constexpr int ra = odd ? 1 : 2, rb = odd ? 2 : 1;  // rounding of even / odd window columns
#pragma unroll
                    for (int j = 0; j < NW; j += 2) {
                        v1[j] = tap<ra>(odd ? bot1[j] : top1[j], cur1[j]), v1[j + 1] = tap<rb>(odd ? bot1[j + 1] : top1[j + 1], cur1[j + 1]);
                        v2[j] = tap<ra>(odd ? bot2[j] : top2[j], cur2[j]), v2[j + 1] = tap<rb>(odd ? bot2[j + 1] : top2[j + 1], cur2[j + 1]);
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < NW; j++) {
                        v1[j] = cur1[j];
                        v2[j] = cur2[j];
                    }
                }
                int c1[8], c2[8];
                if (SX == 2) {
                    int w1[6], w2[6];
#pragma unroll
                    for (int j = 0; j < 6; j++) {
                        w1[j] = v1[j];
                        w2[j] = v2[j];
                    }
                    hfilter2t(w1, c1);
                    hfilter2t(w2, c2);
                } else {
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        c1[j] = v1[j];
                        c2[j] = v2[j];
                    }
                }
#pragma unroll
                for (int x = 0; x < 8; x++) {
                    const int yv = my[(8 * r + x) * TS];
                    int R, G, B;
                    to_rgb<MODE>(yv, c1[x], c2[x], R, G, B);
                    px[3 * x] = R;
                    px[3 * x + 1] = G;
                    px[3 * x + 2] = B;
                }
                if (KB == kStoreCanvas) {
#pragma unroll
                    for (int k = 0; k < 6; k++) wd[k] = pack_sat4(px[4 * k], px[4 * k + 1], px[4 * k + 2], px[4 * k + 3]);
                } else {  // component by component: wd[2 c], wd[2 c + 1] = the eight samples of component c
#pragma unroll
                    for (int c = 0; c < 3; c++) {
                        wd[2 * c] = pack_sat4(px[c], px[3 + c], px[6 + c], px[9 + c]);
                        wd[2 * c + 1] = pack_sat4(px[12 + c], px[15 + c], px[18 + c], px[21 + c]);
                    }
                }
            }
            if constexpr (KB == kStoreRuns || KB == kStoreRunsF) {  // staged in the line's luma slots, which are consumed
                if (valid) {
#pragma unroll
                    for (int k = 0; k < 6; k++) my[(8 * r + k) * NT] = (int)wd[k];
                }
            } else if (KB != kStoreCanvas) {
                if (valid) {
#pragma unroll
                    for (int c = 0; c < 3; c++) store_row<K>(out, c, pl + c, plane_at(pl + c, X, Y + r), wd[2 * c], wd[2 * c + 1], xmax);
                }
            } else if (valid) {
                uint8_t *o = obase + (uint64_t)r * opitch;
                if (xmax == 7 && ((reinterpret_cast<uintptr_t>(o) & 7u) == 0)) {
                    uint2 *o2 = reinterpret_cast<uint2 *>(o);
#pragma unroll
                    for (int k = 0; k < 3; k++) o2[k] = make_uint2(wd[2 * k], wd[2 * k + 1]);
                } else {
#pragma unroll
                    for (int x = 0; x < 8; x++) {
                        if (x <= xmax) {
#pragma unroll
                            for (int i = 3 * x; i < 3 * x + 3; i++) o[i] = (uint8_t)(wd[i >> 2] >> (8 * (i & 3)));
                        }
                    }
                }
            }
        };
        if (SY == 2) {
#pragma unroll 1
            for (int r = 0; r < 8; r += 2) {
                if (r > ymax) break;  // uniform over the warp (same block row)
                one_line(r, std::false_type());
                if (r + 1 <= ymax) one_line(r + 1, std::true_type());
                // advance the line window after every odd output line (upsampler.cpp:160-165)
                if (valid) {
#pragma unroll
                    for (int j = 0; j < NW; j++) {
                        top1[j] = cur1[j];
                        cur1[j] = bot1[j];
                        top2[j] = cur2[j];
                        cur2[j] = bot2[j];
                    }
                }
                if (r < 6) fetch(cy0 + (r >> 1) + 2, bot1, bot2);
            }
        } else {
#pragma unroll 1
            for (int r = 0; r < 8; r++) {
                if (r > ymax) break;
                one_line(r, std::false_type());
                if (r < 7) fetch(cy0 + r + 1, cur1, cur2);
            }
        }
    };
    // one instantiation per colour mode keeps every per-pixel branch out of the line loop
    if (!ycbcr) lines(std::integral_constant<int, 2>());
    else if (wide) lines(std::integral_constant<int, 1>());
    else lines(std::integral_constant<int, 0>());
    if constexpr (KB == kStoreRuns || KB == kStoreRunsF) {
        if (valid) store_staged<K, 3, NT>(out, pl, my, X, Y, xmin, xmax, ymin, ymax);
    }
}

// grid (luma block columns / 32, luma block rows / 4, frames or kWideSlots)
// five CTAs per SM: ptxas fits the kernel into 86 registers without spilling, and 20 resident warps hide the load latency
// better than 16 (six CTAs = 80 registers is slower again)
#ifndef B200JPG_B2_MINCTAS
#define B200JPG_B2_MINCTAS 5
#endif
template <int NC, int SX, int SY, typename T, bool kListed, int K>
__global__ void __launch_bounds__(kThreadsB, B200JPG_B2_MINCTAS)
reconstruct_kernel(const FrameRecon *__restrict__ frames, const int16_t *__restrict__ coef, const T *__restrict__ samples,
                   const uint32_t *__restrict__ wide_flags, const uint32_t *__restrict__ list, StoreDst<K> __restrict__ out) {
    __shared__ int ys[64 * kThreadsB];  // [coefficient][thread]; warps only ever touch their own 32 columns
    if (!kListed) {
        const FrameRecon &f = frames[blockIdx.z];
        reconstruct_tile<NC, SX, SY, T, false, K>(f, ys, coef, samples, 0u, sizeof(T) == 4 && wide_flags[f.status_idx] != 0u, out);
    } else {
        const uint32_t n = list[0];
        for (uint32_t k = blockIdx.z; k < n; k += gridDim.z) {
            const FrameRecon &f = frames[list[1 + k]];
            reconstruct_tile<NC, SX, SY, T, false, K>(f, ys, coef, samples, 0u, sizeof(T) == 4 && wide_flags[f.status_idx] != 0u, out);
            __syncwarp();
        }
    }
}

// B200JPG_FLAG_OUTPUT_RGB: the grey instance of b2 whose rows leave through three descriptors (grey frames have no exact pass)
template <int K>
__global__ void __launch_bounds__(kThreadsB, B200JPG_B2_MINCTAS)
reconstruct_rgb_kernel(const FrameRecon *__restrict__ frames, const int16_t *__restrict__ coef, StoreDst<K> __restrict__ out) {
    __shared__ int ys[64 * kThreadsB];
    reconstruct_tile<1, 1, 1, int16_t, false, K, 1, 3>(frames[blockIdx.z], ys, coef, nullptr, 0u, false, out);
}


// =====================================================================================================
// 4:2:0 frames: chroma IDCT + luma IDCT + upsampling + colour + store in ONE kernel
// =====================================================================================================
// A CTA covers 32 luma block columns x kRows420 luma block rows, one warp per row. Phase 1 fills the chroma window
// (Window420) with the int16 samples of both chroma components:
//  - warps 0 .. kRows420/2 - 1: one chroma block row under the tile each, 16 Cb + 16 Cr blocks through the tile helpers;
//  - the next two warps: the line above / below the tile, the row pass of the chroma block row above / below, then only output
//    row 7 / 0 of the column pass;
//  - every warp: the columns left and right of the tile (corners included), column 7 / 0 of the neighbouring blocks, eight
//    lanes per block: one output of the row pass per coefficient row (a dot product), then one column pass.
// Phase 2 is b2's reconstruct_tile<3, 2, 2> with the chroma window read from shared memory instead of the planes. HBM sees
// coefficients in and pixels out only: b1's chroma planes (written once, read once: 16.6 MB per 4K frame) and the memory
// they take are gone. Window positions outside the chroma plane are never read: phase 2 clamps its addressing to the true
// subsampled size like b2 (upsamplerbase.cpp:322-323, upsampler.cpp:100-106), and the clamped positions lie in the window.
// Range flags as in b1 + b2: a window sample outside int16 flags the frame `narrow`, and the int32 instance (list-driven)
// redoes it; there a window sample beyond +-kWide selects the 64-bit colour mode for the CTA.

// The warp's 32 blocks of coefficients come in as 4 KB of 16-byte pieces, eight per lane (piece i * 32 + lane): a chroma row is
// two runs of 2 KB (Cb blocks 0..15, Cr blocks 16..31). tile_stash parks the pieces in the warp's tile -- the upper half of an
// int32 tile (piece (block, row) at row segment 32 + 4 row + block / 8, slot (block % 8) ^ row: conflict-free both ways), all of
// an int16 one (tile_stash_at) --, tile_idct hands every lane its own block and runs the row pass and the column pass
// (dct/idct.cpp:237-334) as two compact loops over the tile [sample][lane].
template <typename Have>
__device__ __forceinline__ void tile_fetch(uint4 (&pc)[8], const uint4 *__restrict__ src_a, const uint4 *__restrict__ src_b, Have have) {
    const uint32_t lane = threadIdx.x & 31, sub = lane >> 3;
#pragma unroll
    for (uint32_t i = 0; i < 8; i++) {
        const uint4 *p = (i < 4) ? src_a + (i * 32u + lane) : src_b + ((i - 4u) * 32u + lane);
        pc[i] = have(4u * i + sub) ? __ldg(p) : make_uint4(0u, 0u, 0u, 0u);
    }
}

// the byte offset of the pieces in a warp's tile of Y
template <typename Y>
constexpr uint32_t kStash = sizeof(Y) == 2 ? 0u : 4096u;

template <typename Y>
__device__ __forceinline__ void tile_stash(Y *ys, const uint4 (&pc)[8]) {
    tile_stash_at<kStash<Y>>((uint32_t)__cvta_generic_to_shared(ys), pc);
}

// `sink(k, r, a, b)` receives the samples (row r, columns k and k + 1) of this lane's block, k even; only = -1: all 64 samples,
// only = 0 / 7: row 0 / 7 alone. kRows: coefficient rows 0 .. kRows - 1 may be non-zero, the others are zero in every block of
// the warp: their row pass would only yield zeros, so it is skipped and the column pass sees literal zeros (the same integer
// arithmetic, folded by the compiler). Returns in mn / mx (both start at 0) the min / max of what was sunk (int32 tile) or of
// the row-pass outputs (int16 tile: outside int16 they have wrapped; inside, the samples fit int16, see tile_rows16).
template <int kRows, typename Y, typename Sink>
__device__ __forceinline__ void tile_idct_rows(Y *ys, int only, int &mn, int &mx, Sink sink) {
    constexpr bool k16 = sizeof(Y) == 2;
    constexpr int kRound = k16 ? kRound16 : 2048;  // the int16 tile's row pass leaves the level shift to the column pass
    const uint32_t lane = threadIdx.x & 31;
    Y *my = ys + lane;
    if constexpr (k16) {
        tile_rows16<kRows>(ys, mn, mx);
    } else {
        const uint32_t wseg = (uint32_t)__cvta_generic_to_shared(ys);
        const uint32_t mine = wseg + 128u * (32u + (lane >> 3));
        auto piece = [&](int r) { return lds128(mine + 512u * (uint32_t)r + 16u * ((lane & 7u) ^ (uint32_t)r)); };
        uint4 q = piece(0);
#pragma unroll 1
        for (int r = 0; r < kRows; r++) {
            const uint4 qn = piece((r < kRows - 1) ? r + 1 : r);
            int v[8];
            unpack_row_raw(q, v);
            if (r == 0) v[0] = WADD(v[0], 128 << 3);  // dcoffset << 3 (idct.cpp:233,244), the << 4 preshift left out like in the inputs
            idct8t<16, 5>(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
            __syncwarp();
#pragma unroll
            for (int k = 0; k < 8; k++) my[(8 * r + k) * 32] = v[k];
            q = qn;
        }
        mx = 0, mn = 0;
    }
#pragma unroll 1
    for (int k = 0; k < 8; k += 2) {
        int a[8], b[8];
#pragma unroll
        for (int r = 0; r < 8; r++) {
            a[r] = (r < kRows) ? (int)my[(8 * r + k) * 32] : 0;
            b[r] = (r < kRows) ? (int)my[(8 * r + k + 1) * 32] : 0;
        }
        if (only < 0) {
            idct8t<kRound, 12>(a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7]);
            idct8t<kRound, 12>(b[0], b[1], b[2], b[3], b[4], b[5], b[6], b[7]);
#pragma unroll
            for (int r = 0; r < 8; r++) sink(k, r, a[r], b[r]);
            if constexpr (!k16) {
#pragma unroll
                for (int r = 0; r < 8; r += 2) {
                    mx = __vimax3_s32(__vimax3_s32(mx, a[r], a[r + 1]), b[r], b[r + 1]);
                    mn = __vimin3_s32(__vimin3_s32(mn, a[r], a[r + 1]), b[r], b[r + 1]);
                }
            }
        } else {
            // output 0 / 7 of the column pass is one dot product: the butterfly of idct8t is linear in front of its rounding shift
            //   out0 = 512 v0 + 710 v1 + 669 v2 + 602 v3 + 512 v4 + 402 v5 + 277 v6 + 141 v7,  out7 = the same with the odd terms negated
            auto one = [&](const int (&v)[8]) {
                const int even = WADD(WADD(WMUL(v[0], 512), WMUL(v[2], 669)), WADD(WMUL(v[4], 512), WMUL(v[6], 277)));
                const int odd = WADD(WADD(WMUL(v[1], 710), WMUL(v[3], 602)), WADD(WMUL(v[5], 402), WMUL(v[7], 141)));
                return WADD(only == 0 ? WADD(even, odd) : WSUB(even, odd), kRound) >> 12;
            };
            const int sa = one(a), sb = one(b);
            sink(k, only, sa, sb);
            if constexpr (!k16) {
                mx = __vimax3_s32(mx, sa, sb);
                mn = __vimin3_s32(mn, sa, sb);
            }
        }
    }
}

// Chroma blocks of ordinary images rarely carry anything in coefficient rows 6 and 7 (4:2:0 q75 frames of the benchmark: in
// about 98 % of the warps none of the 32 blocks does), so the warp checks once and takes the shorter instance when it can.
template <typename Y, typename Sink>
__device__ __forceinline__ void tile_idct(Y *ys, int only, int &mn, int &mx, Sink sink) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t mine = (uint32_t)__cvta_generic_to_shared(ys) + kStash<Y> + 128u * (lane >> 3);
    const uint4 p6 = lds128(mine + 512u * 6u + 16u * ((lane & 7u) ^ 6u)), p7 = lds128(mine + 512u * 7u + 16u * ((lane & 7u) ^ 7u));
    const bool high = ((p6.x | p6.y | p6.z | p6.w) | (p7.x | p7.y | p7.z | p7.w)) != 0u;
    if (__any_sync(0xffffffffu, high)) tile_idct_rows<8>(ys, only, mn, mx, sink);
    else tile_idct_rows<6>(ys, only, mn, mx, sink);
}

template <typename T, int K>
__device__ __forceinline__ void reconstruct420_tile(const FrameRecon &f, Tile420<T, K> *ys, uint32_t win, const int16_t *__restrict__ coef,
                                                    uint32_t *__restrict__ narrow_flags, StoreDst<K> __restrict__ out) {
    using Wn = Window420<T>;
    using Y = Tile420<T, K>;
    constexpr int kHalf = kRows420 / 2;  // chroma block rows under the tile
    constexpr bool kClip = kClipKind<K>;  // a cropped frame: tile (tx0, ty0) + blockIdx, past the clip rectangle nothing
    const uint32_t vbw = ((kClip ? f.clip_x1 : f.width) + 7) >> 3, vbh = ((kClip ? f.clip_y1 : f.height) + 7) >> 3;
    const uint32_t tile_x = kClip ? f.tx0 + blockIdx.x : blockIdx.x, tile_y = kClip ? f.ty0 + blockIdx.y : blockIdx.y;
    if (tile_x * 32u >= vbw || tile_y * (uint32_t)kRows420 >= vbh) return;  // whole CTA
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int bwc = (int)f.bw[1], bhc = (int)f.bh[1];
    const int cbx0 = 16 * (int)tile_x, cby0 = kHalf * (int)tile_y;
    auto at = [&](uint32_t comp, int line, int col) {
        return win + comp * (uint32_t)Wn::kCompBytes + (uint32_t)line * (uint32_t)Wn::kLineBytes + (uint32_t)col * (uint32_t)sizeof(T);
    };
    int mn = 0, mx = 0;

    // ---- phase 1a: chroma block rows -> window; q = the block row relative to the tile (-1: the row above, kHalf: below)
    if (warp < (uint32_t)kHalf + 2u) {
        const int q = (warp < (uint32_t)kHalf) ? (int)warp : (warp == (uint32_t)kHalf ? -1 : kHalf);
        const int cby = cby0 + q;
        if (cby >= 0 && cby < bhc) {
            Y *yw = ys + warp * 2048u;  // this warp's 8 KB (int16 tile: 4 KB) of the luma tile, free until phase 2
            uint4 pc[8];
            const uint4 *src_a = reinterpret_cast<const uint4 *>(coef + f.coef_base[1] + ((uint64_t)cby * (uint32_t)bwc + (uint32_t)cbx0) * 64u);
            const uint4 *src_b = reinterpret_cast<const uint4 *>(coef + f.coef_base[2] + ((uint64_t)cby * (uint32_t)bwc + (uint32_t)cbx0) * 64u);
            tile_fetch(pc, src_a, src_b, [&](uint32_t blk) { return cbx0 + (int)(blk & 15u) < bwc; });
            tile_stash(yw, pc);
            const uint32_t comp = lane >> 4;
            const int col = 4 + 8 * (int)(lane & 15u), line0 = 1 + 8 * q;  // window line of the block's row 0
            tile_idct(yw, q < 0 ? 7 : (q == kHalf ? 0 : -1), mn, mx,
                      [&](int k, int r, int a, int b) { win_store2<T>(at(comp, line0 + r, col + k), a, b); });
        }
    }
    // ---- phase 1b: the columns left / right of the tile. Eight lanes per (block row j, component, side); lane r&7 = coefficient
    // row r, then = output row r of the column pass
    {
        const uint32_t job = threadIdx.x >> 3, r = lane & 7u;
        if (job < 4u * (kHalf + 2)) {  // warp-uniform: four jobs per warp
            const uint32_t side = job & 1u, hc = (job >> 1) & 1u;
            const int j = (int)(job >> 2), cby = cby0 - 1 + j;
            const int nb = side ? cbx0 + 16 : cbx0 - 1;
            const bool exists = nb >= 0 && nb < bwc && cby >= 0 && cby < bhc;
            int v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            if (exists) unpack_row_raw(__ldg(reinterpret_cast<const uint4 *>(coef + f.coef_base[1 + hc] + ((uint64_t)cby * (uint32_t)bwc + (uint32_t)nb) * 64u) + r), v);
            if (r == 0) v[0] = WADD(v[0], 128 << 3);
            // output 0 (side 1) / 7 (side 0) of the row pass, the dot products of tile_idct
            const int even = WADD(WADD(WMUL(v[0], 512), WMUL(v[2], 669)), WADD(WMUL(v[4], 512), WMUL(v[6], 277)));
            const int odd = WADD(WADD(WMUL(v[1], 710), WMUL(v[3], 602)), WADD(WMUL(v[5], 402), WMUL(v[7], 141)));
            const int inter = WADD(side ? WADD(even, odd) : WSUB(even, odd), 16) >> 5;  // row pass without the << 4 preshift, see unpack_row_raw
            int c[8];
#pragma unroll
            for (int i = 0; i < 8; i++) c[i] = __shfl_sync(0xffffffffu, inter, (int)((lane & ~7u) + (uint32_t)i));
            idct8t<2048, 12>(c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[7]);
            int s = c[0];
#pragma unroll
            for (int i = 1; i < 8; i++) s = (r == (uint32_t)i) ? c[i] : s;
            const int line = 8 * j - 7 + (int)r;  // the row above contributes its row 7 only, the row below its row 0
            if (exists && line >= 0 && line < Wn::kLines) {
                win_store<T>(at(hc, line, side ? 132 : 3), s);
                mx = s > mx ? s : mx;
                mn = s < mn ? s : mn;
            }
        }
    }
    // int16: a window sample (int32 tile) or a row-pass output of phase 1a (int16 tile) or a sample of phase 1b outside int16
    const bool out_of_range = (sizeof(T) == 2) ? (mx > 32767 || mn < -32768) : (mx > kWide || mn < -kWide);
    const bool flagged = __syncthreads_or(out_of_range) != 0;
    if (sizeof(T) == 2 && flagged && threadIdx.x == 0) atomicOr(narrow_flags + f.status_idx, 1u);  // `narrow`: the int32 instance redoes the frame

    // ---- phase 2: the luma rows
    reconstruct_tile<3, 2, 2, T, true, K, 1, 3, Y>(f, ys, coef, nullptr, win, sizeof(T) == 4 && flagged, out, narrow_flags);
}

// Resident warps per SM that reconstruct420_kernel<T, ..., K> is compiled for (__launch_bounds__). The CTA is latency-bound:
// 16 warps instead of 20 made it 21 % slower (DESIGN §4). With the 16-bit tile (Canvas, Planar) six CTAs = 24 warps fit, at 80
// registers without spills; the other int16 kinds stay at five (20 warps, 96 registers): the float kinds spill at 80, and the
// strided store, one byte per instruction, was 16 % slower at six CTAs (DESIGN §9). The int32 instance (rare frames) keeps 12,
// which keeps it free of spills. (-DB200JPG_R420_WARPS16=20: the 16-bit tile at five CTAs, for comparisons.)
#ifndef B200JPG_R420_WARPS16
#define B200JPG_R420_WARPS16 24
#endif
template <typename T, int K>
constexpr int kWarps420 = sizeof(T) == 4 ? 12 : (sizeof(Tile420<T, K>) == 2 ? B200JPG_R420_WARPS16 : 20);

// grid (luma block columns / 32, luma block rows / kRows420, frames or kWideSlots); dynamic shared memory
// Window420<T, Tile420<T, K>>::kSmemBytes
template <typename T, bool kListed, int K>
__global__ void __launch_bounds__(kThreads420, kWarps420<T, K> / kRows420)
reconstruct420_kernel(const FrameRecon *__restrict__ frames, const int16_t *__restrict__ coef, uint32_t *__restrict__ narrow_flags,
                      const uint32_t *__restrict__ list, StoreDst<K> __restrict__ out) {
    using Y = Tile420<T, K>;
    extern __shared__ __align__(16) uint8_t smem420[];
    Y *ys = reinterpret_cast<Y *>(smem420);  // phase 2: the luma tile; phase 1: 8 KB (int16 tile: 4 KB) per warp
    const uint32_t win = (uint32_t)__cvta_generic_to_shared(smem420) + (uint32_t)Window420<T, Y>::kYsBytes;
    if (!kListed) {
        reconstruct420_tile<T, K>(frames[blockIdx.z], ys, win, coef, narrow_flags, out);
    } else {
        const uint32_t n = list[0];
        for (uint32_t k = blockIdx.z; k < n; k += gridDim.z) {
            reconstruct420_tile<T, K>(frames[list[1 + k]], ys, win, coef, narrow_flags, out);
            __syncthreads();  // the next frame's phase 1 overwrites the tile and the window
        }
    }
}


// ---- 8-bit 4:2:0 frames downscaled by KS (B200JPG_FLAG_DOWNSCALE_k): reconstruct420_kernel's tile on the reduced frame ------
// The CTA covers 32 x kRows420 blocks of the REDUCED frame (f.width x f.height). Phase 1 fills the int32 chroma window (the same
// Window420 lines and columns, now of the reduced chroma planes) straight from the chroma coefficients: every coefficient block
// whose (8/KS) x (8/KS) samples meet the window goes through scaled_idct_block once, and the samples that lie in the window and in
// the plane (f.cw x f.ch) are stored. Phase 2 is reconstruct_tile<3, 2, 2, int32_t, true, K, KS>: luma from the KS x KS
// coefficient blocks under each output block, then the same upsampling, colour transformation and stores as every other 4:2:0
// frame. No sample planes; a window sample beyond +-kWide selects the 64-bit colour mode for the CTA, as in the int32 instance
// of reconstruct420_kernel.
template <int KS, int K>
__global__ void __launch_bounds__(kThreads420, 12 / kRows420)
reconstruct420_scaled_kernel(const FrameRecon *__restrict__ frames, const int16_t *__restrict__ coef, StoreDst<K> __restrict__ out) {
    using Wn = Window420<int32_t>;
    constexpr int N = 8 / KS;
    extern __shared__ __align__(16) uint8_t smem420s[];
    int *ys = reinterpret_cast<int *>(smem420s);
    const uint32_t win = (uint32_t)__cvta_generic_to_shared(smem420s) + (uint32_t)Wn::kYsBytes;
    const FrameRecon &f = frames[blockIdx.z];
    constexpr bool kClip = kClipKind<K>;  // a cropped frame: tile (tx0, ty0) + blockIdx, past the clip rectangle nothing
    const uint32_t vbw = ((kClip ? f.clip_x1 : f.width) + 7) >> 3, vbh = ((kClip ? f.clip_y1 : f.height) + 7) >> 3;
    const uint32_t tile_x = kClip ? f.tx0 + blockIdx.x : blockIdx.x, tile_y = kClip ? f.ty0 + blockIdx.y : blockIdx.y;
    if (tile_x * 32u >= vbw || tile_y * (uint32_t)kRows420 >= vbh) return;  // whole CTA
    const int cw = (int)f.cw, ch = (int)f.ch;
    const int wy0 = 4 * kRows420 * (int)tile_y - 1, wx0 = 128 * (int)tile_x - 4;  // window line 0 / column 0
    // the window positions that lie in the plane: lines y0..y1, columns x0..x1 (columns 3..132 of the window)
    const int y0 = max(wy0, 0), y1 = min(wy0 + Wn::kLines - 1, ch - 1), x0 = max(wx0 + 3, 0), x1 = min(wx0 + 132, cw - 1);
    int mn = 0, mx = 0;
    if (y0 <= y1 && x0 <= x1) {
        const int by0 = y0 / N, bx0 = x0 / N, nby = y1 / N - by0 + 1, nbx = x1 / N - bx0 + 1;
        const uint32_t bwc = f.coef_bw[1];
        for (int job = (int)threadIdx.x; job < 2 * nby * nbx; job += kThreads420) {
            const int comp = job / (nby * nbx), rest = job - comp * nby * nbx;
            const int cy = by0 + rest / nbx, cx = bx0 + rest % nbx;
            int sm[N][N];
            scaled_idct_block<KS>(coef + f.coef_base[1 + comp] + ((uint64_t)cy * bwc + (uint32_t)cx) * 64u, 128 << 4, sm);
#pragma unroll
            for (int n = 0; n < N; n++) {
#pragma unroll
                for (int m = 0; m < N; m++) {
                    const int y = N * cy + n, x = N * cx + m;
                    if (y >= y0 && y <= y1 && x >= x0 && x <= x1) {
                        sts32(win + (uint32_t)comp * (uint32_t)Wn::kCompBytes + (uint32_t)(y - wy0) * (uint32_t)Wn::kLineBytes + (uint32_t)(x - wx0) * 4u,
                              sm[n][m]);
                        mx = max(mx, sm[n][m]);
                        mn = min(mn, sm[n][m]);
                    }
                }
            }
        }
    }
    const bool wide = __syncthreads_or(mx > kWide || mn < -kWide) != 0;
    reconstruct_tile<3, 2, 2, int32_t, true, K, KS>(f, ys, coef, nullptr, win, wide, out);
}

// =====================================================================================================
// generic reconstruction: any number of components (1..4), any subsampling factors (1..4, per component)
// =====================================================================================================
// The formats outside the tuned kernels -- chroma factors 3 and 4, components with different factors, a subsampled first
// component, two or four components (SURVEY 8f4) -- are rare, so this path is written for exactness, not for speed: every
// component goes through idct_planes_kernel into an int32 sample plane, then one thread per 8x8 OUTPUT block follows
// Upsampler<sx,sy>::UpsampleRegion to the letter (upsampling/upsampler.cpp:83-112, VerticalFilterCore<1..4> :114-268,
// HorizontalFilterCore<1..4> :270-386 -- including the in-place stores of the horizontal cores, whose order is part of the
// result) and the colour transformation in 64 bits (ycbcrtrafo.cpp:842-850 / identity numerics.hpp:69).
__device__ __forceinline__ int gmix(int a, int wa, int b, int wb, int rnd, int sh) {
    return (int)((unsigned)wa * (unsigned)a + (unsigned)wb * (unsigned)b + (unsigned)rnd) >> sh;
}

// one 8x8 block of component samples at output position (X, Y), upsampled by (sx, sy); plane = IDCT output, pitch in samples,
// (w, h) = true subsampled size; edge replication dest[-1] = dest[0], dest[w] = dest[w-1] (upsamplerbase.cpp:322-323) by clamping
__device__ void generic_upsample_block(const int32_t *__restrict__ plane, uint32_t pitch, int w, int h, int sx, int sy, int X, int Y, int *out) {
    const int y = Y / sy;
    const int x0 = X / sx - ((sx > 1) ? 1 : 0);
    int top = (y > 0) ? y - 1 : y, cur = y, bot = (y + 1 < h) ? y + 1 : y;
    int ymod = Y % sy;
    const int xmod = X % sx;
    auto at = [&](int x, int yy) { return plane[(size_t)yy * pitch + (size_t)clampi(x, 0, w - 1)]; };
    for (int row = 0; row < 8; row++) {
        int *o = out + 8 * row;
        int advance = 0;
        if (sy == 1) {
            for (int j = 0; j < 8; j++) o[j] = at(x0 + j, cur);
            if (cur + 1 < h) cur++;
        } else if (sy == 2) {
            const int nb = (ymod == 0) ? top : bot;
            for (int j = 0; j < 8; j++) o[j] = gmix(at(x0 + j, nb), 1, at(x0 + j, cur), 3, ((j & 1) == ymod) ? 2 : 1, 2);
            advance = (ymod == 1);
        } else if (sy == 3) {
            if (ymod == 1) {
                for (int j = 0; j < 8; j++) o[j] = at(x0 + j, cur);
            } else {
                const int nb = (ymod == 0) ? top : bot;
                for (int j = 0; j < 8; j++) o[j] = gmix(at(x0 + j, nb), 1, at(x0 + j, cur), 3, (((j & 1) == 0) == (ymod == 0)) ? 2 : 1, 2);
            }
            advance = (ymod == 2);
        } else {
            const int nb = (ymod < 2) ? top : bot;
            const bool far = (ymod == 0 || ymod == 3);  // far from the sample line: weights 3:5, else 1:7
            for (int j = 0; j < 8; j++) {
                int rnd;
                if (ymod == 0 || ymod == 2 || ymod == 3) rnd = (j & 1) ? 3 : 4;
                else rnd = (j & 1) ? 4 : 3;
                o[j] = gmix(at(x0 + j, nb), far ? 3 : 1, at(x0 + j, cur), far ? 5 : 7, rnd, 3);
            }
            advance = (ymod == 3);
        }
        if (sy > 1) {
            if (advance) {
                ymod = 0;
                top = cur;
                cur = bot;
                if (bot + 1 < h) bot++;
            } else {
                ymod++;
            }
        }
        // horizontal, in place, in the reference's store order (src[i] = o[i + 1])
        if (sx == 2) {
            int *src = o + 1, t;
            o[7] = gmix(src[4], 1, src[3], 3, 1, 2);
            o[6] = gmix(src[2], 1, src[3], 3, 2, 2);
            o[5] = gmix(src[3], 1, src[2], 3, 1, 2);
            o[4] = gmix(src[1], 1, src[2], 3, 2, 2);
            o[3] = gmix(src[2], 1, src[1], 3, 1, 2);
            o[2] = gmix(src[0], 1, src[1], 3, 2, 2);
            t = src[0];
            o[1] = gmix(src[1], 1, t, 3, 1, 2);  // src[1] is the NEW o[2]
            o[0] = gmix(src[-1], 1, t, 3, 2, 2);
        } else if (sx == 3) {
            int *src = o + 1, t;
            if (xmod == 0) {
                o[7] = src[2];
                o[6] = gmix(src[1], 1, src[2], 3, 2, 2);
                o[5] = gmix(src[2], 1, src[1], 3, 1, 2);
                o[4] = src[1];
                o[3] = gmix(src[0], 1, src[1], 3, 2, 2);
                o[2] = gmix(src[1], 1, src[0], 3, 1, 2);
                o[0] = gmix(src[-1], 1, src[0], 3, 2, 2);
                o[1] = src[0];
            } else if (xmod == 1) {
                o[7] = gmix(src[3], 1, src[2], 3, 1, 2);
                o[6] = src[2];
                o[5] = gmix(src[1], 1, src[2], 3, 2, 2);
                o[4] = gmix(src[2], 1, src[1], 3, 1, 2);
                o[3] = src[1];
                t = src[0];
                o[2] = gmix(t, 1, src[1], 3, 2, 2);
                o[1] = gmix(src[1], 1, t, 3, 1, 2);
                o[0] = t;
            } else {
                o[7] = gmix(src[2], 1, src[3], 3, 2, 2);
                o[6] = gmix(src[3], 1, src[2], 3, 1, 2);
                o[5] = src[2];
                o[4] = gmix(src[1], 1, src[2], 3, 2, 2);
                o[3] = gmix(src[2], 1, src[1], 3, 1, 2);
                o[2] = src[1];
                t = src[0];
                o[1] = gmix(t, 1, src[1], 3, 2, 2);
                o[0] = gmix(src[1], 1, t, 3, 1, 2);
            }
        } else if (sx == 4) {
            int *src = o + 1, t;
            o[7] = gmix(src[2], 3, src[1], 5, 1, 3);
            o[6] = gmix(src[2], 1, src[1], 7, 2, 3);
            o[5] = gmix(src[0], 1, src[1], 7, 1, 3);
            o[4] = gmix(src[0], 3, src[1], 5, 2, 3);
            t = src[0];
            o[3] = gmix(src[1], 3, t, 5, 1, 3);
            o[2] = gmix(src[1], 1, t, 7, 2, 3);
            o[1] = gmix(src[-1], 1, t, 7, 1, 3);
            o[0] = gmix(src[-1], 3, t, 5, 2, 3);
        }
    }
}

// grid (output block columns / 64, output block rows, frames). K: kStoreCanvas, or kStoreStrided / kStoreStridedF for every
// described destination (this path stores one sample at a time anyway); with kStoreClip (cropped frames) the grid covers the
// tiles of kGenericTileBlocks x 1 blocks from (tx0, ty0) on, and only samples inside the clip rectangle are stored

// B200JPG_FLAG_OUTPUT_* (MODE = OutMode, described kinds only): the clamped samples w[0 .. nc) of pixel (x, y) as the frame's output
// components. Luma: L = (19595 w0 + 38470 w1 + 7471 w2 + 32768) >> 16 (PIL's convert("L"), libjpeg's rgb_gray_convert; below 2^31 for
// 12-bit samples too) into component 0; Replicate: w0 into components 0, 1 and 2, each with its own component's map. CmykRgb /
// CmykLuma: w[0 .. 3) is the frame's RGB (cmyk_to_rgb), stored as three components / as L like Luma
template <int K, int MODE>
__device__ __forceinline__ void store_mode_pixel(StoreDst<K> out, uint32_t status_idx, int x, int y, const int (&w)[4], bool deep) {
    constexpr int KB = kBaseKind<K>;
    static_assert(KB == kStoreStrided || KB == kStoreStridedF, "output modes store through descriptors");
    constexpr bool kL = MODE == (int)OutMode::Luma || MODE == (int)OutMode::CmykLuma;
    constexpr bool kRgb = MODE == (int)OutMode::CmykRgb;  // w[0 .. 3) is already the RGB of the frame (cmyk_to_rgb)
    const int v = kL ? (19595 * w[0] + 38470 * w[1] + 7471 * w[2] + 32768) >> 16 : w[0];
    constexpr uint32_t no = kL ? 1u : 3u;
#pragma unroll
    for (uint32_t c = 0; c < no; c++) {
        const int u = kRgb ? w[c] : v;
        if constexpr (KB == kStoreStridedF) {
            store_elem(out.type, plane_at(out.planes + 4u * status_idx + c, x, y), map_int(table_of<kTableKind<K>>(out), c, u, pick4(out.scale, c), pick4(out.bias, c)));
        } else {
            uint8_t *o = plane_at(out + 4u * status_idx + c, x, y);
            if (deep) *reinterpret_cast<uint16_t *>(o) = (uint16_t)u;
            else *o = (uint8_t)u;
        }
    }
}

// MODE (OutMode): Coded, or for the groups of an output mode (B200JPG_FLAG_OUTPUT_RGB / _L) Luma, Replicate, CmykRgb or CmykLuma,
// K then kStoreStrided or kStoreStridedF, with or without the clip
template <int K, int MODE = (int)OutMode::Coded>
__global__ void __launch_bounds__(64)
generic_reconstruct_kernel(const FrameRecon *__restrict__ frames, const int32_t *__restrict__ samples, StoreDst<K> __restrict__ out) {
    constexpr int KB = kBaseKind<K>;
    constexpr bool kClip = kClipKind<K>;
    constexpr bool kCmyk = MODE == (int)OutMode::CmykRgb || MODE == (int)OutMode::CmykLuma;  // 8-bit four-component frames only
    const FrameRecon &f = frames[blockIdx.z];
    // (a CMYK / YCCK group's frames all have four components: a constant count keeps the per-component arrays in registers)
    const uint32_t W = f.width, H = f.height, nc = kCmyk ? 4u : f.ncomp;
    const uint32_t bx = (kClip ? f.tx0 * kGenericTileBlocks : 0u) + blockIdx.x * 64 + threadIdx.x, by = (kClip ? f.ty0 : 0u) + blockIdx.y;
    if (bx >= (W + 7) / 8 || by >= (H + 7) / 8) return;
    if (kClip && (bx < f.clip_x0 / 8 || bx >= (f.clip_x1 + 7) / 8 || by < f.clip_y0 / 8 || by >= (f.clip_y1 + 7) / 8)) return;
    const int X = 8 * (int)bx, Y = 8 * (int)by;
    // 64 upsampled samples per subsampled component (local memory: this path is not tuned); a component at full resolution is
    // read where it lies -- inside the image its sample plane IS the upsampled image
    int buf[4][64];
    const int32_t *direct[4] = {nullptr, nullptr, nullptr, nullptr};
    for (uint32_t c = 0; c < nc; c++) {
        const int sx = f.csx[c], sy = f.csy[c];
        const int w = (int)((W + sx - 1) / sx), h = (int)((H + sy - 1) / sy);
        if (sx == 1 && sy == 1) direct[c] = samples + f.sample_base[c] + (uint64_t)Y * (8u * f.bw[c]) + (uint64_t)X;
        else generic_upsample_block(samples + f.sample_base[c], 8u * f.bw[c], w, h, sx, sy, X, Y, buf[c]);
    }
    auto base_at = [&](uint32_t c, int x, int y) -> int { return direct[c] ? direct[c][(uint64_t)y * (8u * f.bw[c]) + (uint32_t)x] : buf[c][8 * y + x]; };
    int xmax = (X + 7 < (int)W) ? 7 : (int)((W - 1) & 7), ymax = (Y + 7 < (int)H) ? 7 : (int)((H - 1) & 7), xmin = 0, ymin = 0;
    if constexpr (kClip) {
        xmin = max((int)f.clip_x0 - X, 0), xmax = min((int)f.clip_x1 - 1 - X, xmax);
        ymin = max((int)f.clip_y0 - Y, 0), ymax = min((int)f.clip_y1 - 1 - Y, ymax);
    }
    if (!kCmyk && (f.xt & 1u)) {  // (a four-component frame is never a JPEG XT frame: parse_codestream refuses it)
        // ---- JPEG XT (SURVEY 8f3): base image + residual image, YCbCrTrafo<..., Residual | Extended | ClampFlag, ...>::YCbCr2RGB
        // colortrafo/ycbcrtrafo.cpp:747-880 with the tables of the 8-bit integer profile (colortransformerfactory.cpp:300-352,
        // 425-520; ParametricToneMappingBox::ScaledTableOf boxes/parametrictonemappingbox.cpp:387-426): Q = identity over the
        // pre-shifted range 0..4095, R2 = floor(i / 16 + 0.5), L = identity over 0..255, C = identity; a lookup clamps its index
        int rbuf[3][64];
        const int32_t *rdirect[3] = {nullptr, nullptr, nullptr};
        for (uint32_t c = 0; c < nc; c++) {
            const int sx = f.res_csx[c], sy = f.res_csy[c];
            const int w = (int)((W + sx - 1) / sx), h = (int)((H + sy - 1) / sy);
            if (sx == 1 && sy == 1) rdirect[c] = samples + f.res_sample_base[c] + (uint64_t)Y * (8u * f.res_bw[c]) + (uint64_t)X;
            else generic_upsample_block(samples + f.res_sample_base[c], 8u * f.res_bw[c], w, h, sx, sy, X, Y, rbuf[c]);
        }
        auto res_at = [&](uint32_t c, int x, int y) -> int { return rdirect[c] ? rdirect[c][(uint64_t)y * (8u * f.res_bw[c]) + (uint32_t)x] : rbuf[c][8 * y + x]; };
        auto clamp_to = [](long long v, long long mx) { return v < 0 ? 0ll : (v > mx ? mx : v); };
        for (int y = ymin; y <= ymax; y++) {
            uint8_t *o = nullptr;
            if constexpr (KB == kStoreCanvas) o = out + f.out_base + ((uint64_t)(Y + y) * W + (uint64_t)X) * nc;
            for (int x = xmin; x <= xmax; x++) {
                const int i = 8 * y + x;
                long long res[3] = {128, 128, 128}, v[3] = {0, 0, 0};
                if (nc == 3 && (f.xt & 4u)) {  // the residual: Q table, R transformation (FIX_COLOR_TO_INTCOLOR), R2 table
                    const long long yv = clamp_to(res_at(0, x, y), 4095), cb = clamp_to(res_at(1, x, y), 4095) - (128 << 4), cr = clamp_to(res_at(2, x, y), 4095) - (128 << 4);
                    res[0] = (yv * 8192 + cr * 11485 + 4096) >> 13;
                    res[1] = (yv * 8192 - cb * 2819 - cr * 5850 + 4096) >> 13;
                    res[2] = (yv * 8192 + cb * 14516 + 4096) >> 13;
                } else {
                    for (uint32_t c = 0; c < nc; c++) res[c] = clamp_to(res_at(c, x, y), 4095);
                }
                if (nc == 3 && (f.xt & 2u)) {  // the base image: L transformation (FIX_COLOR_TO_INT), L table
                    const long long yv = base_at(0, x, y), cb = (long long)base_at(1, x, y) - (128 << 4), cr = (long long)base_at(2, x, y) - (128 << 4);
                    v[0] = (yv * 8192 + cr * 11485 + 65536) >> 17;
                    v[1] = (yv * 8192 - cb * 2819 - cr * 5850 + 65536) >> 17;
                    v[2] = (yv * 8192 + cb * 14516 + 65536) >> 17;
                } else {
                    for (uint32_t c = 0; c < nc; c++) v[c] = ((long long)base_at(c, x, y) + 8) >> 4;
                }
                if constexpr (MODE != (int)OutMode::Coded) {
                    int w[4] = {0, 0, 0, 0};
                    for (uint32_t c = 0; c < nc; c++) w[c] = (int)clamp_to(clamp_to(v[c], 255) + ((clamp_to(res[c], 4095) + 8) >> 4) - 128, 255);
                    store_mode_pixel<K, MODE>(out, f.status_idx, X + x, Y + y, w, false);
                    continue;
                }
                for (uint32_t c = 0; c < nc; c++) {  // merge and clamp (:863-878, :935-947)
                    const uint8_t m = (uint8_t)clamp_to(clamp_to(v[c], 255) + ((clamp_to(res[c], 4095) + 8) >> 4) - 128, 255);
                    if constexpr (KB == kStoreCanvas) o[nc * x + c] = m;
                    else if constexpr (KB == kStoreStridedF)
                        store_elem(out.type, plane_at(out.planes + 4u * f.status_idx + c, X + x, Y + y), map_int(table_of<kTableKind<K>>(out), c, m, pick4(out.scale, c), pick4(out.bias, c)));
                    else *plane_at(out + 4u * f.status_idx + c, X + x, Y + y) = m;
                }
            }
        }
        return;
    }
    // level shift, chroma offset and clamp scale with the precision; 12-bit frames leave as native-endian 16-bit samples
    // (what the reference writes into CTYP_UWORD bitmaps)
    const bool deep = f.precision > 8;
    const long long maxval = (1ll << f.precision) - 1, coff = 16ll << (f.precision - 1u);
    for (int y = ymin; y <= ymax; y++) {
        const uint64_t at = ((uint64_t)(Y + y) * W + (uint64_t)X) * nc;
        uint8_t *o8 = nullptr;
        uint16_t *o16 = nullptr;
        if constexpr (KB == kStoreCanvas) {
            o8 = out + f.out_base + at;
            o16 = reinterpret_cast<uint16_t *>(out + f.out_base) + at;
        }
        for (int x = xmin; x <= xmax; x++) {
            long long v[4];
            if (nc == 3 && f.ycbcr) {
                const long long yv = base_at(0, x, y), cb = (long long)base_at(1, x, y) - coff, cr = (long long)base_at(2, x, y) - coff;
                v[0] = (yv * 8192 + cr * 11485 + 65536) >> 17;
                v[1] = (yv * 8192 - cb * 2819 - cr * 5850 + 65536) >> 17;
                v[2] = (yv * 8192 + cb * 14516 + 65536) >> 17;
            } else {
                for (uint32_t c = 0; c < nc; c++) v[c] = ((long long)base_at(c, x, y) + 8) >> 4;
            }
            if constexpr (MODE != (int)OutMode::Coded) {
                int w[4] = {0, 0, 0, 0};
                for (uint32_t c = 0; c < nc; c++) w[c] = (int)(v[c] < 0 ? 0 : (v[c] > maxval ? maxval : v[c]));
                if constexpr (kCmyk) cmyk_to_rgb(w, f.ycck != 0);
                store_mode_pixel<K, MODE>(out, f.status_idx, X + x, Y + y, w, deep);
                continue;
            }
            for (uint32_t c = 0; c < nc; c++) {
                const long long w = v[c] < 0 ? 0 : (v[c] > maxval ? maxval : v[c]);
                if constexpr (KB == kStoreCanvas) {
                    if (deep) o16[nc * x + c] = (uint16_t)w;
                    else o8[nc * x + c] = (uint8_t)w;
                } else if constexpr (KB == kStoreStridedF) {
                    store_elem(out.type, plane_at(out.planes + 4u * f.status_idx + c, X + x, Y + y), map_int(table_of<kTableKind<K>>(out), c, (int)w, pick4(out.scale, c), pick4(out.bias, c)));
                } else {
                    uint8_t *o = plane_at(out + 4u * f.status_idx + c, X + x, Y + y);
                    if (deep) *reinterpret_cast<uint16_t *>(o) = (uint16_t)w;
                    else *o = (uint8_t)w;
                }
            }
        }
    }
}

// B200JPG_FLAG_NO_UPSAMPLE: component blockIdx.z of frame blockIdx.y, one thread per sample of its true (subsampled) size:
// COLOR_TO_INT and the clamp of the identity transformation (tools/numerics.hpp:69), nothing else. K as for
// generic_reconstruct_kernel
template <int K>
__global__ void __launch_bounds__(256)
planes_out_kernel(const FrameRecon *__restrict__ frames, const int32_t *__restrict__ samples, StoreDst<K> __restrict__ out) {
    const FrameRecon &f = frames[blockIdx.y];
    const uint32_t c = blockIdx.z;
    if (c >= f.ncomp) return;
    uint64_t before = 0;  // samples of the planes in front of this one
    for (uint32_t k = 0; k < c; k++) before += (uint64_t)((f.width + f.csx[k] - 1) / f.csx[k]) * ((f.height + f.csy[k] - 1) / f.csy[k]);
    const uint32_t w = (f.width + f.csx[c] - 1) / f.csx[c], h = (f.height + f.csy[c] - 1) / f.csy[c];
    const int maxval = (1 << f.precision) - 1;
    for (uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x; i < (uint64_t)w * h; i += (uint64_t)gridDim.x * 256) {
        const uint32_t x = (uint32_t)(i % w), y = (uint32_t)(i / w);
        int v = (samples[f.sample_base[c] + (uint64_t)y * (8u * f.bw[c]) + x] + 8) >> 4;
        v = v < 0 ? 0 : (v > maxval ? maxval : v);
        if constexpr (K == kStoreCanvas) {
            if (f.precision > 8) reinterpret_cast<uint16_t *>(out + f.out_base)[before + i] = (uint16_t)v;
            else out[f.out_base + before + i] = (uint8_t)v;
        } else if constexpr (kBaseKind<K> == kStoreStridedF) {
            store_elem(out.type, plane_at(out.planes + 4u * f.status_idx + c, (int)x, (int)y), map_int(table_of<kTableKind<K>>(out), c, v, pick4(out.scale, c), pick4(out.bias, c)));
        } else {
            uint8_t *o = plane_at(out + 4u * f.status_idx + c, (int)x, (int)y);
            if (f.precision > 8) *reinterpret_cast<uint16_t *>(o) = (uint16_t)v;
            else *o = (uint8_t)v;
        }
    }
}

}  // namespace

// the destination argument of a launch of kind K
template <int K>
static StoreDst<K> dst_of(const ReconLaunch &l) {
    if constexpr (K == kStoreCanvas) {
        return l.out;
    } else if constexpr (kFloatKind<K>) {
        FloatDst d{};
        d.planes = l.planes;
        d.type = l.convert->type;
        for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++) d.scale[c] = l.convert->scale[c], d.bias[c] = l.convert->bias[c];
        d.table = l.table;
        return d;
    } else {
        return l.planes;
    }
}

template <typename T, bool kListed, int K>
static void launch_b2(const ReconLaunch &l, dim3 grid, const T *samples, cudaStream_t s) {
    const StoreDst<K> out = dst_of<K>(l);
    if constexpr (!kListed && K != kStoreCanvas) {
        if (l.mode == OutMode::Replicate) {
            reconstruct_rgb_kernel<K><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, out);
            return;
        }
    }
    if (l.ncomp == 1) {
        reconstruct_kernel<1, 1, 1, T, kListed, K><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, samples, l.wide_flags, l.narrow_list, out);
    } else if (l.subx == 2 && l.suby == 1) {
        reconstruct_kernel<3, 2, 1, T, kListed, K><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, samples, l.wide_flags, l.narrow_list, out);
    } else if (l.subx == 1 && l.suby == 2) {
        reconstruct_kernel<3, 1, 2, T, kListed, K><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, samples, l.wide_flags, l.narrow_list, out);
    } else {
        reconstruct_kernel<3, 1, 1, T, kListed, K><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, samples, l.wide_flags, l.narrow_list, out);
    }
}

template <int K>
static int launch_recon420(const ReconLaunch &l, cudaStream_t s, int *launches) {
    const uint32_t gx = (l.max_bw0 + 31) / 32, gy = (l.max_bh0 + kRows420 - 1) / kRows420;
    constexpr int smem16 = Window420<int16_t, Tile420<int16_t, K>>::kSmemBytes, smem32 = Window420<int32_t>::kSmemBytes;
    cudaError_t e = cudaFuncSetAttribute(reconstruct420_kernel<int16_t, false, K>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e == cudaSuccess && smem16 > 48 * 1024) e = cudaFuncSetAttribute(reconstruct420_kernel<int16_t, false, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem16);
    if (e == cudaSuccess && smem32 > 48 * 1024) e = cudaFuncSetAttribute(reconstruct420_kernel<int32_t, true, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem32);
    if (e != cudaSuccess) return (int)e;
    reconstruct420_kernel<int16_t, false, K><<<dim3(gx, gy, l.n_frames), kThreads420, smem16, s>>>(l.frames, l.coef, l.narrow_flags, nullptr, dst_of<K>(l));
    // the exact pass over the frames flagged `narrow` (none for real images: two near-empty launches)
    narrow_list_kernel<<<1, 256, 0, s>>>(l.frames, l.n_frames, l.narrow_flags, l.narrow_list);
    reconstruct420_kernel<int32_t, true, K><<<dim3(gx, gy, kWideSlots), kThreads420, smem32, s>>>(l.frames, l.coef, l.narrow_flags, l.narrow_list, dst_of<K>(l));
    if (launches) *launches = 3;
    return (int)cudaGetLastError();
}

// 8-bit 4:2:0 frames downscaled by l.downscale: one launch of reconstruct420_scaled_kernel
template <int K, int KS>
static int launch_recon420_scaled_k(const ReconLaunch &l, cudaStream_t s, int *launches) {
    const uint32_t gx = (l.max_bw0 + 31) / 32, gy = (l.max_bh0 + kRows420 - 1) / kRows420;
    constexpr int smem = Window420<int32_t>::kSmemBytes;
    cudaError_t e = cudaFuncSetAttribute(reconstruct420_scaled_kernel<KS, K>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e == cudaSuccess && smem > 48 * 1024) e = cudaFuncSetAttribute(reconstruct420_scaled_kernel<KS, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return (int)e;
    reconstruct420_scaled_kernel<KS, K><<<dim3(gx, gy, l.n_frames), kThreads420, smem, s>>>(l.frames, l.coef, dst_of<K>(l));
    if (launches) *launches = 1;
    return (int)cudaGetLastError();
}

template <int K>
static int launch_recon420_scaled(const ReconLaunch &l, cudaStream_t s, int *launches) {
    if (l.downscale == 2) return launch_recon420_scaled_k<K, 2>(l, s, launches);
    if (l.downscale == 4) return launch_recon420_scaled_k<K, 4>(l, s, launches);
    return launch_recon420_scaled_k<K, 8>(l, s, launches);
}

template <int K>
static int launch_recon_generic(const ReconLaunch &l, cudaStream_t s, int *launches) {
    uint32_t mb = 0;
    mb = l.max_bwc * l.max_bhc;  // the largest component block grid of the group (set by the host for generic groups)
    const uint32_t cblocks = (mb + kThreadsB - 1) / kThreadsB;
    int n = 0;
    if (l.generic_phase != 2) {
        const dim3 grid(cblocks, l.n_frames, l.ncomp);
        if (l.path == ReconPath::Generic) idct_planes_kernel<int32_t, false><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, l.samples32, l.wide_flags, nullptr, 0);
        else if (l.downscale == 2) idct_scaled_planes_kernel<2><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, l.samples32);
        else if (l.downscale == 4) idct_scaled_planes_kernel<4><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, l.samples32);
        else idct_scaled_planes_kernel<8><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, l.samples32);
        n++;
    }
    if (l.generic_phase == 1) {
        if (launches) *launches = n;
        return (int)cudaGetLastError();
    }
    n++;
    if (l.planes_out) {  // never cropped (b200jpg_batch_create_crop refuses B200JPG_FLAG_NO_UPSAMPLE with a rectangle)
        if constexpr (!kClipKind<K>) {
            const uint32_t gx = std::min<uint32_t>((l.max_bw0 * l.max_bh0 * 64u + 255u) / 256u, 4096u);
            planes_out_kernel<K><<<dim3(gx, l.n_frames, l.ncomp), 256, 0, s>>>(l.frames, l.samples32, dst_of<K>(l));
        }
    } else {
        const dim3 grid((l.max_bw0 + kGenericTileBlocks - 1) / kGenericTileBlocks, l.max_bh0, l.n_frames);
        bool done = false;  // an output mode's group (never the canvas: its slots are described)
        if constexpr (K != kStoreCanvas) {
            if (l.mode == OutMode::Luma) generic_reconstruct_kernel<K, (int)OutMode::Luma><<<grid, 64, 0, s>>>(l.frames, l.samples32, dst_of<K>(l));
            if (l.mode == OutMode::Replicate) generic_reconstruct_kernel<K, (int)OutMode::Replicate><<<grid, 64, 0, s>>>(l.frames, l.samples32, dst_of<K>(l));
            if (l.mode == OutMode::CmykRgb) generic_reconstruct_kernel<K, (int)OutMode::CmykRgb><<<grid, 64, 0, s>>>(l.frames, l.samples32, dst_of<K>(l));
            if (l.mode == OutMode::CmykLuma) generic_reconstruct_kernel<K, (int)OutMode::CmykLuma><<<grid, 64, 0, s>>>(l.frames, l.samples32, dst_of<K>(l));
            done = l.mode != OutMode::Coded;
        }
        if (!done) generic_reconstruct_kernel<K><<<grid, 64, 0, s>>>(l.frames, l.samples32, dst_of<K>(l));
    }
    if (launches) *launches = n;
    return (int)cudaGetLastError();
}

template <int K>
static int launch_recon_kind(const ReconLaunch &l, cudaStream_t s, int *launches) {
    if (l.path == ReconPath::Turbo || l.path == ReconPath::TurboGeneric) {  // (every frame of such a group is cropped: admit_crops)
        if constexpr (kClipKind<K>) return launch_turbo<(kFloatKind<K> ? kStoreStridedF : kStoreStrided) | kStoreClip | (K & kStoreTable)>(l, s, launches);
        return (int)cudaErrorInvalidValue;
    }
    if (l.path == ReconPath::Generic || l.path == ReconPath::Scaled)
        return launch_recon_generic<K == kStoreCanvas ? kStoreCanvas : ((kFloatKind<K> ? kStoreStridedF : kStoreStrided) | (K & (kStoreClip | kStoreTable)))>(l, s, launches);
    if (l.path == ReconPath::Fused420) return launch_recon420<K>(l, s, launches);
    if (l.path == ReconPath::Scaled420) return launch_recon420_scaled<K>(l, s, launches);
    int n = 0;  // ReconPath::Tiled
    const uint32_t cblocks = (l.max_bwc * l.max_bhc + kThreadsB - 1) / kThreadsB;
    const uint32_t gx = (l.max_bw0 + 31) / 32, gy = (l.max_bh0 + kThreadsB / 32 - 1) / (kThreadsB / 32);
    // every frame through the int16 planes, B200JPG_RECON_CHUNK frames at a time (0: all at once): in chunks the planes b1 writes
    // are still in L2 when b2 reads them
    uint32_t chunk = l.n_frames;
    if (const char *e = getenv("B200JPG_RECON_CHUNK")) {
        const long v = atol(e);
        if (v > 0 && (uint32_t)v < chunk) chunk = (uint32_t)v;
    }
    for (uint32_t f0 = 0; f0 < l.n_frames; f0 += chunk) {
        const uint32_t nf = (l.n_frames - f0 < chunk) ? (l.n_frames - f0) : chunk;
        ReconLaunch c = l;
        c.frames = l.frames + f0;
        if (l.ncomp > 1) {
            if constexpr (kClipKind<K>)  // cropped frames: the chroma blocks their tiles read (FrameRecon::cb_*)
                idct_planes_crop_kernel<int16_t, false><<<dim3(cblocks, nf, l.ncomp - 1), kThreadsB, 0, s>>>(c.frames, l.coef, l.samples16, l.narrow_flags, nullptr, 1);
            else
                idct_planes_kernel<int16_t, false><<<dim3(cblocks, nf, l.ncomp - 1), kThreadsB, 0, s>>>(c.frames, l.coef, l.samples16, l.narrow_flags, nullptr, 1);
            n++;
        }
        launch_b2<int16_t, false, K>(c, dim3(gx, gy, nf), l.samples16, s);
        n++;
    }
    // the exact pass over the frames that were flagged `narrow` (none for real images: three near-empty launches)
    if (l.ncomp > 1) {
        narrow_list_kernel<<<1, 256, 0, s>>>(l.frames, l.n_frames, l.narrow_flags, l.narrow_list);
        if constexpr (kClipKind<K>)  // the exact pass recomputes the same chroma blocks
            idct_planes_crop_kernel<int32_t, true><<<dim3(cblocks, kWideSlots, l.ncomp - 1), kThreadsB, 0, s>>>(l.frames, l.coef, l.samples32, l.wide_flags, l.narrow_list, 1);
        else
            idct_planes_kernel<int32_t, true><<<dim3(cblocks, kWideSlots, l.ncomp - 1), kThreadsB, 0, s>>>(l.frames, l.coef, l.samples32, l.wide_flags, l.narrow_list, 1);
        launch_b2<int32_t, true, K>(l, dim3(gx, gy, kWideSlots), l.samples32, s);
        n += 3;
    }
    if (launches) *launches = n;
    return (int)cudaGetLastError();
}

// the destination kind is chosen per group from the descriptors (b200jpg_batch_decode_into), never by the caller
int launch_recon(const ReconLaunch &l, void *stream, int *launches) {
    cudaStream_t s = (cudaStream_t)stream;
    if (!l.planes) return launch_recon_kind<kStoreCanvas>(l, s, launches);
    if (l.convert && l.table) {  // (b200jpg_batch_decode_into_table)
        if (l.clip) return launch_recon_kind<kStoreRunsF | kStoreClip | kStoreTable>(l, s, launches);
        if (l.runs) return launch_recon_kind<kStoreRunsF | kStoreTable>(l, s, launches);
        return l.planar ? launch_recon_kind<kStorePlanarF | kStoreTable>(l, s, launches) : launch_recon_kind<kStoreStridedF | kStoreTable>(l, s, launches);
    }
    if (l.clip) return l.convert ? launch_recon_kind<kStoreRunsF | kStoreClip>(l, s, launches) : launch_recon_kind<kStoreRuns | kStoreClip>(l, s, launches);
    if (l.runs) return l.convert ? launch_recon_kind<kStoreRunsF>(l, s, launches) : launch_recon_kind<kStoreRuns>(l, s, launches);
    if (l.convert) return l.planar ? launch_recon_kind<kStorePlanarF>(l, s, launches) : launch_recon_kind<kStoreStridedF>(l, s, launches);
    if (l.planar) return launch_recon_kind<kStorePlanar>(l, s, launches);
    return launch_recon_kind<kStoreStrided>(l, s, launches);
}

}  // namespace b200jpg
