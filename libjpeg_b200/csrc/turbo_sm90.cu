// turbo_sm90.cu -- B200JPG_FLAG_LIBJPEG_TURBO (DESIGN §16): libjpeg-turbo's reconstruction on sm_90a, in a translation unit of
// its own so that no instance of recon_sm100.cu changes.
//
//   turbo_idct_kernel          one lane per 8x8 block: JDCT_ISLOW (C form, 64-bit intermediates) and the post-IDCT range-limit
//                              table -> one uint8 plane per component (ReconPath::TurboGeneric: every component of the frame;
//                              ReconPath::Turbo: the chroma blocks under the frame's clip tiles and their halo)
//   turbo_reconstruct_kernel   ReconPath::Turbo (grey, 4:4:4, 4:2:2, 4:4:0, 4:2:0 with full-resolution luma): a tile of 32 x 4
//                              luma blocks, luma IDCT'd into shared memory, chroma read from the planes, upsampled, converted and
//                              stored pixel by pixel along x
//   turbo_generic_kernel       ReconPath::TurboGeneric: one thread per output pixel from the planes of every component
//   turbo_*_draft_kernel       the same three for drafted frames (DESIGN §17, groups of ReconLaunch::downscale > 1): each block
//                              leaves the IDCT as FrameRecon::idct[c]^2 samples (islow, jpeg_idct_4x4, jpeg_idct_2x2 or
//                              jpeg_idct_1x1), the Turbo tile holds luma blocks of S = 8 / k, and the planes are upsampled by the
//                              ratios after the IDCT
//   turbo_cmyk_*kernel         turbo_generic_kernel and its draft form for the 8-bit Adobe CMYK / YCCK frames of an output mode
//                              (DESIGN §18): four components read, Pillow's conversion (cmyk_sm90.cuh), three or one stored
// Every frame of a flagged batch is cropped (abi.cpp: admit_crops), so both kinds store through described destinations with
// the clip.
#include <cuda_runtime.h>

#include <type_traits>

#include "cmyk_sm90.cuh"
#include "internal.hpp"
#include "store_sm90.cuh"

namespace b200jpg {
namespace {

// int32 is exact for a pass while every sum it forms stays inside int32. As a linear form of the pass's 8 inputs no sum of the
// butterfly has an L1 norm above 61214 (tests/test_turbo_cpu.py finds it by brute force over sign patterns), so pass 1 is exact for
// |F| <= (2^31 - 1 - 2^10) / 61214 = 35081 -- every int16 coefficient of the store -- and pass 2 while every pass-1 result has
// |v| <= (2^31 - 1 - 2^17) / 61214 = 35079; a block with a larger pass-1 result runs pass 2 in 64 bits
constexpr int kPass1Exact = 35081, kPass2Exact = 35079;
static_assert(kPass1Exact >= 32768, "pass 1 takes the int16 coefficients in int32");

// one 8-point islow pass over d[0 .. 8), in place: outputs (x + 2^(shift - 1)) >> shift, T = int or long long
template <typename T, int kShift>
__device__ __forceinline__ void islow8(T (&d)[8]) {
    // even part
    T z1 = (d[2] + d[6]) * (T)4433;
    const T tmp2 = z1 + d[6] * (T)-15137, tmp3 = z1 + d[2] * (T)6270;
    const T tmp0 = (d[0] + d[4]) * (T)8192, tmp1 = (d[0] - d[4]) * (T)8192;
    const T t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
    // odd part
    T o0 = d[7], o1 = d[5], o2 = d[3], o3 = d[1];
    z1 = o0 + o3;
    T z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3;
    const T z5 = (z3 + z4) * (T)9633;
    o0 *= (T)2446, o1 *= (T)16819, o2 *= (T)25172, o3 *= (T)12299;
    z1 *= (T)-7373, z2 *= (T)-20995, z3 *= (T)-16069, z4 *= (T)-3196;
    z3 += z5, z4 += z5;
    o0 += z1 + z3, o1 += z2 + z4, o2 += z2 + z3, o3 += z1 + z4;
    constexpr T r = (T)1 << (kShift - 1);
    d[0] = (t10 + o3 + r) >> kShift, d[7] = (t10 - o3 + r) >> kShift;
    d[1] = (t11 + o2 + r) >> kShift, d[6] = (t11 - o2 + r) >> kShift;
    d[2] = (t12 + o1 + r) >> kShift, d[5] = (t12 - o1 + r) >> kShift;
    d[3] = (t13 + o0 + r) >> kShift, d[4] = (t13 - o0 + r) >> kShift;
}

// pass kShift over the 8 lines of s (columns when kCols), through T
template <typename T, int kShift, bool kCols>
__device__ __forceinline__ void islow_pass(int (&s)[8][8]) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
        T d[8];
#pragma unroll
        for (int j = 0; j < 8; j++) d[j] = kCols ? (T)s[j][k] : (T)s[k][j];
        islow8<T, kShift>(d);
#pragma unroll
        for (int j = 0; j < 8; j++) (kCols ? s[j][k] : s[k][j]) = (int)d[j];
    }
}

// the post-IDCT range-limit table at v & 1023: 0..127 -> v + 128, 128..511 -> 255, 512..895 -> 0, 896..1023 -> v - 896
__device__ __forceinline__ uint32_t range_limit(int v) {
    const int i = v & 1023;
    return (uint32_t)(i < 128 ? i + 128 : (i < 512 ? 255 : (i < 896 ? 0 : i - 896)));
}

// one block: its 64 dequantised coefficients at src -> 8 rows of 8 samples at dst (row pitch `pitch`, 8-byte aligned)
__device__ __forceinline__ void turbo_idct_block(const int16_t *__restrict__ coef, uint8_t *dst, uint32_t pitch) {
    int s[8][8];
    const uint4 *src = reinterpret_cast<const uint4 *>(coef);
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const uint4 q = __ldg(src + r);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int k = 0; k < 4; k++) {
            s[r][2 * k] = (int)(int16_t)(w[k] & 0xffffu);
            s[r][2 * k + 1] = (int)w[k] >> 16;
        }
    }
    islow_pass<int, 11, true>(s);
    int mx = 0;
#pragma unroll
    for (int r = 0; r < 8; r++)
#pragma unroll
        for (int k = 0; k < 8; k++) mx = max(mx, abs(s[r][k]));
    if (mx <= kPass2Exact) islow_pass<int, 18, false>(s);
    else islow_pass<long long, 18, false>(s);
#pragma unroll
    for (int r = 0; r < 8; r++) {
        uint2 w;
        w.x = range_limit(s[r][0]) | range_limit(s[r][1]) << 8 | range_limit(s[r][2]) << 16 | range_limit(s[r][3]) << 24;
        w.y = range_limit(s[r][4]) | range_limit(s[r][5]) << 8 | range_limit(s[r][6]) << 16 | range_limit(s[r][7]) << 24;
        *reinterpret_cast<uint2 *>(dst + (uint64_t)r * pitch) = w;
    }
}

// jpeg_idct_4x4 / jpeg_idct_2x2 (jidctred.c). As for islow, int32 is exact for a pass while every sum stays inside int32: as a
// linear form of the pass's inputs no sum has an L1 norm above 77910 (4x4) or 85759 (2x2) (tests/test_draft_cpu.py finds both by
// brute force), so pass 1 (rounding 2^11 / 2^12) is exact for |F| <= 27563 / 25040 and pass 2 (2^18 / 2^19) for pass-1 results
// |v| <= 27560 / 25034. int16 coefficients exceed the pass-1 bounds: a block runs each pass in 64 bits when its inputs do
constexpr int kRed4Pass1Exact = 27563, kRed4Pass2Exact = 27560, kRed2Pass1Exact = 25040, kRed2Pass2Exact = 25034;

// one line of jpeg_idct_4x4 over d[0 .. 8) (d[4] unused) -> 4 outputs (x + 2^(kShift - 1)) >> kShift
template <typename T, int kShift>
__device__ __forceinline__ void red4(const T (&d)[8], T (&o)[4]) {
    const T t0 = d[0] * (T)16384, t2 = d[2] * (T)15137 + d[6] * (T)-6270;
    const T t10 = t0 + t2, t12 = t0 - t2;
    const T o0 = d[7] * (T)-1730 + d[5] * (T)11893 + d[3] * (T)-17799 + d[1] * (T)8697;
    const T o2 = d[7] * (T)-4176 + d[5] * (T)-4926 + d[3] * (T)7373 + d[1] * (T)20995;
    constexpr T r = (T)1 << (kShift - 1);
    o[0] = (t10 + o2 + r) >> kShift, o[3] = (t10 - o2 + r) >> kShift;
    o[1] = (t12 + o0 + r) >> kShift, o[2] = (t12 - o0 + r) >> kShift;
}

// one line of jpeg_idct_2x2 over d[0 .. 8) (d[2], d[4], d[6] unused) -> 2 outputs
template <typename T, int kShift>
__device__ __forceinline__ void red2(const T (&d)[8], T (&o)[2]) {
    const T t10 = d[0] * (T)32768;
    const T t0 = d[7] * (T)-5906 + d[5] * (T)6967 + d[3] * (T)-10426 + d[1] * (T)29692;
    constexpr T r = (T)1 << (kShift - 1);
    o[0] = (t10 + t0 + r) >> kShift, o[1] = (t10 - t0 + r) >> kShift;
}

// the inputs an S-point reduced line reads: 4 x 4 skips index 4, 2 x 2 every even index but 0
template <int S>
__device__ __forceinline__ constexpr bool red_input(int k) {
    return k != 4 && !(S == 2 && (k == 2 || k == 6));
}

// pass 1 of the S-point reduced IDCT (S = 4, 2): the columns of s the second pass reads -> the S rows of ws
template <int S, typename T>
__device__ __forceinline__ void red_pass1(const int (&s)[8][8], int (&ws)[S][8]) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
        if (!red_input<S>(k)) continue;
        T d[8], o[S];
#pragma unroll
        for (int j = 0; j < 8; j++) d[j] = (T)s[j][k];
        if constexpr (S == 4) red4<T, 12>(d, o);
        else red2<T, 13>(d, o);
#pragma unroll
        for (int j = 0; j < S; j++) ws[j][k] = (int)o[j];
    }
}

// pass 2 along the S rows of ws -> S x S samples at dst (row pitch `pitch`)
template <int S, typename T>
__device__ __forceinline__ void red_pass2(const int (&ws)[S][8], uint8_t *dst, uint32_t pitch) {
#pragma unroll
    for (int r = 0; r < S; r++) {
        T d[8], o[S];
#pragma unroll
        for (int j = 0; j < 8; j++) d[j] = red_input<S>(j) ? (T)ws[r][j] : (T)0;
        if constexpr (S == 4) {
            red4<T, 19>(d, o);
            *reinterpret_cast<uint32_t *>(dst + (uint64_t)r * pitch) =
                range_limit((int)o[0]) | range_limit((int)o[1]) << 8 | range_limit((int)o[2]) << 16 | range_limit((int)o[3]) << 24;
        } else {
            red2<T, 20>(d, o);
            *reinterpret_cast<uint16_t *>(dst + (uint64_t)r * pitch) = (uint16_t)(range_limit((int)o[0]) | range_limit((int)o[1]) << 8);
        }
    }
}

// one block at the reduced size S (4 or 2): its 64 dequantised coefficients -> S rows of S samples at dst (S-byte aligned); each pass
// in int32 when the block's inputs to it are inside that pass's bound, else in 64 bits
template <int S>
__device__ __forceinline__ void turbo_idct_block_reduced(const int16_t *__restrict__ coef, uint8_t *dst, uint32_t pitch) {
    constexpr int kB1 = S == 4 ? kRed4Pass1Exact : kRed2Pass1Exact, kB2 = S == 4 ? kRed4Pass2Exact : kRed2Pass2Exact;
    int s[8][8];
    const uint4 *src = reinterpret_cast<const uint4 *>(coef);
    int mx = 0;
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const uint4 q = __ldg(src + r);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int k = 0; k < 4; k++) {
            s[r][2 * k] = (int)(int16_t)(w[k] & 0xffffu);
            s[r][2 * k + 1] = (int)w[k] >> 16;
            mx = max(mx, max(abs(s[r][2 * k]), abs(s[r][2 * k + 1])));
        }
    }
    int ws[S][8];
    if (mx <= kB1) red_pass1<S, int>(s, ws);
    else red_pass1<S, long long>(s, ws);
    mx = 0;
#pragma unroll
    for (int r = 0; r < S; r++)
#pragma unroll
        for (int k = 0; k < 8; k++)
            if (red_input<S>(k)) mx = max(mx, abs(ws[r][k]));
    if (mx <= kB2) red_pass2<S, int>(ws, dst, pitch);
    else red_pass2<S, long long>(ws, dst, pitch);
}

// grid (blocks / 128, frames, components - first): block t of component first + blockIdx.z of frame blockIdx.y -> 8 x 8 bytes of its
// plane. kRange (ReconPath::Turbo, first = 1): t runs over the chroma blocks [cb_x0, cb_x1) x [cb_y0, cb_y1) only. kDraft (drafted
// groups, turbo_idct_draft_kernel): S x S bytes, S = FrameRecon::idct[c], into a plane of pitch S bw
template <bool kRange, bool kDraft>
__device__ __forceinline__ void turbo_idct(const FrameRecon *__restrict__ frames, const int16_t *__restrict__ coef, uint8_t *__restrict__ planes) {
    const FrameRecon &f = frames[blockIdx.y];
    const uint32_t c = (kRange ? 1u : 0u) + blockIdx.z;
    uint32_t t = blockIdx.x * kThreadsB + threadIdx.x;
    if (c >= f.ncomp) return;
    const uint32_t bw = f.bw[c], bh = f.bh[c];
    if constexpr (kRange) {
        const uint32_t rw = f.cb_x1 - f.cb_x0, rh = f.cb_y1 - f.cb_y0;
        if (t >= rw * rh) return;
        t = (f.cb_y0 + t / rw) * bw + f.cb_x0 + t % rw;
    }
    if (t >= bw * bh) return;
    const uint32_t bx = t % bw, by = t / bw;
    const int16_t *src = coef + f.coef_base[c] + (uint64_t)t * 64u;
    if constexpr (kDraft) {
        const uint32_t S = f.idct[c], pitch = S * bw;
        uint8_t *dst = planes + f.sample_base[c] + (uint64_t)(S * by) * pitch + S * bx;
        if (S == 8) turbo_idct_block(src, dst, pitch);
        else if (S == 4) turbo_idct_block_reduced<4>(src, dst, pitch);
        else if (S == 2) turbo_idct_block_reduced<2>(src, dst, pitch);
        else *dst = (uint8_t)range_limit((src[0] + 4) >> 3);  // jpeg_idct_1x1
    } else {
        const uint32_t pitch = 8u * bw;
        turbo_idct_block(src, planes + f.sample_base[c] + (uint64_t)(8u * by) * pitch + 8u * bx, pitch);
    }
}

template <bool kRange>
__global__ void __launch_bounds__(kThreadsB)
turbo_idct_kernel(const FrameRecon *__restrict__ frames, const int16_t *__restrict__ coef, uint8_t *__restrict__ planes) {
    turbo_idct<kRange, false>(frames, coef, planes);
}

template <bool kRange>
__global__ void __launch_bounds__(kThreadsB)
turbo_idct_draft_kernel(const FrameRecon *__restrict__ frames, const int16_t *__restrict__ coef, uint8_t *__restrict__ planes) {
    turbo_idct<kRange, true>(frames, coef, planes);
}

// sample (x, y) of the frame-size image of a component whose plane p (row pitch `pitch`, real size w x h) is upsampled by the
// integer factors fx x fy: h2v1 / h2v2 fancy for w > 2, h1v2 fancy, every other ratio replicated; the row above the first and
// below row h - 1 is that row itself. fancy = false (a frame drafted at 1/8) replicates every ratio
__device__ __forceinline__ int turbo_upsampled(const uint8_t *__restrict__ p, uint32_t pitch, int fx, int fy, int w, int h, int x, int y,
                                               bool fancy = true) {
    auto at = [&](int r, int col) -> int { return __ldg(p + (uint64_t)r * pitch + (uint32_t)col); };
    if (fx == 1 && fy == 1) return at(y, x);
    if (!fancy) return at(y / fy, x / fx);
    const bool odd_y = (y & 1) != 0, odd_x = (x & 1) != 0;
    if (fx == 1 && fy == 2) {  // h1v2
        const int i = y >> 1;
        const int far = at(odd_y ? min(i + 1, h - 1) : max(i - 1, 0), x);
        return (3 * at(i, x) + far + (odd_y ? 2 : 1)) >> 2;
    }
    if (fx != 2 || fy > 2 || w <= 2) return at(y / fy, x / fx);
    const int j = x >> 1, jn = odd_x ? j + 1 : j - 1;
    const bool edge = odd_x ? j == w - 1 : j == 0;
    if (fy == 1) {  // h2v1
        const int a = at(y, j);
        return edge ? a : (3 * a + at(y, jn) + (odd_x ? 2 : 1)) >> 2;
    }
    const int i = y >> 1, ifar = odd_y ? min(i + 1, h - 1) : max(i - 1, 0);  // h2v2
    const int cs = 3 * at(i, j) + at(ifar, j);
    if (edge) return (4 * cs + (odd_x ? 7 : 8)) >> 4;
    return (3 * cs + 3 * at(i, jn) + at(ifar, jn) + (odd_x ? 7 : 8)) >> 4;
}

template <int K>
using TurboDst = std::conditional_t<kFloatKind<K>, FloatDst, const b200jpg_plane *>;

// YCbCr -> RGB (rule 3), clamped, in place
__device__ __forceinline__ void turbo_ycc_rgb(int (&v)[3]) {
    const int yy = v[0], b = v[1] - 128, r = v[2] - 128;
    v[0] = min(max(yy + ((91881 * r + 32768) >> 16), 0), 255);
    v[1] = min(max(yy + ((-22554 * b - 46802 * r + 32768) >> 16), 0), 255);
    v[2] = min(max(yy + ((116130 * b + 32768) >> 16), 0), 255);
}

constexpr int kTurboTileW = 32, kTurboTileH = kThreadsB / 32;  // luma blocks per tile (recon_tile(ReconPath::Turbo))

// grid (tile columns, tile rows, frames) over the tiles from (tx0, ty0) on, kThreadsB threads. Phase 1: thread (lane, warp) IDCTs
// luma block (32 tx + lane, 4 ty + warp) into the shared tile when it meets the clip rectangle. Phase 2: the tile's pixels, 128
// consecutive x per step: luma from the tile, chroma (NC == 3) upsampled by SX x SY from the planes, rule 3, the mode (a
// launch-uniform OutMode, as for turbo_generic_kernel), the store through the frame's descriptors, read once per thread.
// S: the luma block's IDCT size, 8 (turbo_reconstruct_kernel) or that of a drafted frame, 4, 2, 1 (turbo_reconstruct_draft_kernel,
// DESIGN §17): a tile is then 32 S x 4 S output pixels, the chroma planes have pitch FrameRecon::idct[c] bw[c], SX x SY are the
// ratios after the chroma IDCT, and S == 1 (1/8) replicates
template <int NC, int S, int SX, int SY, int K>
__device__ __forceinline__ void turbo_reconstruct(const FrameRecon *__restrict__ frames, const int16_t *__restrict__ coef,
                                                  const uint8_t *__restrict__ planes, int mode, TurboDst<K> out) {
    static_assert(kClipKind<K> && (kBaseKind<K> == kStoreStrided || kBaseKind<K> == kStoreStridedF), "described, cropped destinations");
    constexpr int TW = S * kTurboTileW, TH = S * kTurboTileH;
    __shared__ __align__(16) uint8_t tile[TH * TW];
    const FrameRecon &f = frames[blockIdx.z];
    const int X0 = (int)((f.tx0 + blockIdx.x) * TW), Y0 = (int)((f.ty0 + blockIdx.y) * TH);
    const int cx0 = (int)f.clip_x0, cx1 = (int)f.clip_x1, cy0 = (int)f.clip_y0, cy1 = (int)f.clip_y1;
    if (X0 >= cx1 || Y0 >= cy1) return;  // (uniform over the CTA) a tile beyond this frame's clip range
    {
        const int lane = (int)threadIdx.x & 31, row = (int)threadIdx.x >> 5;
        const int bx = X0 / S + lane, by = Y0 / S + row;
        if (S * bx < cx1 && S * bx + S > cx0 && S * by < cy1 && S * by + S > cy0) {
            const int16_t *src = coef + f.coef_base[0] + ((uint64_t)by * f.bw[0] + (uint32_t)bx) * 64u;
            if constexpr (S == 8) turbo_idct_block(src, tile + 8 * row * TW + 8 * lane, TW);
            else if constexpr (S == 1) tile[row * TW + lane] = (uint8_t)range_limit((__ldg(src) + 4) >> 3);  // jpeg_idct_1x1
            else turbo_idct_block_reduced<S>(src, tile + S * row * TW + S * lane, TW);
        }
    }
    __syncthreads();
    constexpr int kMaxOut = 3;
    uint64_t data[kMaxOut];
    int64_t bpr[kMaxOut];
    int bpp[kMaxOut];
    const uint32_t no = mode == (int)OutMode::Luma ? 1u : (mode == (int)OutMode::Replicate ? 3u : (uint32_t)NC);
#pragma unroll
    for (uint32_t c = 0; c < kMaxOut; c++) {
        data[c] = 0, bpr[c] = 0, bpp[c] = 0;
        if (c >= no) continue;
        const b200jpg_plane *d;
        if constexpr (kFloatKind<K>) d = out.planes + 4u * f.status_idx + c;
        else d = out + 4u * f.status_idx + c;
        asm volatile("ld.global.nc.u64 %0, [%1];" : "=l"(data[c]) : "l"(&d->data));
        asm volatile("ld.global.nc.s32 %0, [%1];" : "=r"(bpp[c]) : "l"(&d->bytes_per_pixel));
        asm volatile("ld.global.nc.s64 %0, [%1];" : "=l"(bpr[c]) : "l"(&d->bytes_per_row));
    }
    const int xa = max(cx0 - X0, 0), xb = min(cx1 - X0, TW), ya = max(cy0 - Y0, 0), yb = min(cy1 - Y0, TH);
    for (int p = (int)threadIdx.x; p < TW * TH; p += kThreadsB) {
        const int lx = p % TW, ly = p / TW;
        if (lx < xa || lx >= xb || ly < ya || ly >= yb) continue;
        const int x = X0 + lx, y = Y0 + ly;
        int v[3];
        v[0] = tile[ly * TW + lx];
        v[1] = v[2] = v[0];
        if constexpr (NC == 3 && S == 8) {
            v[1] = turbo_upsampled(planes + f.sample_base[1], 8u * f.bw[1], SX, SY, (int)f.cw, (int)f.ch, x, y);
            v[2] = turbo_upsampled(planes + f.sample_base[2], 8u * f.bw[2], SX, SY, (int)f.cw, (int)f.ch, x, y);
        } else if constexpr (NC == 3) {
            v[1] = turbo_upsampled(planes + f.sample_base[1], f.idct[1] * f.bw[1], SX, SY, (int)f.cw, (int)f.ch, x, y, S != 1);
            v[2] = turbo_upsampled(planes + f.sample_base[2], f.idct[2] * f.bw[2], SX, SY, (int)f.cw, (int)f.ch, x, y, S != 1);
        }
        if constexpr (NC == 3) {
            if (f.ycbcr) turbo_ycc_rgb(v);
            if (mode == (int)OutMode::Luma) v[0] = (19595 * v[0] + 38470 * v[1] + 7471 * v[2] + 32768) >> 16;
        }
#pragma unroll
        for (uint32_t c = 0; c < kMaxOut; c++) {
            if (c >= no) break;
            uint8_t *o = reinterpret_cast<uint8_t *>(data[c] + (uint64_t)((int64_t)x * bpp[c]) + (uint64_t)((int64_t)y * bpr[c]));
            if constexpr (kFloatKind<K>) store_elem(out.type, o, map_int(table_of<kTableKind<K>>(out), c, v[c], pick4(out.scale, c), pick4(out.bias, c)));
            else *o = (uint8_t)v[c];
        }
    }
}

template <int NC, int SX, int SY, int K>
__global__ void __launch_bounds__(kThreadsB)
turbo_reconstruct_kernel(const FrameRecon *__restrict__ frames, const int16_t *__restrict__ coef, const uint8_t *__restrict__ planes,
                         int mode, TurboDst<K> out) {
    turbo_reconstruct<NC, 8, SX, SY, K>(frames, coef, planes, mode, out);
}

template <int NC, int S, int SX, int SY, int K>
__global__ void __launch_bounds__(kThreadsB)
turbo_reconstruct_draft_kernel(const FrameRecon *__restrict__ frames, const int16_t *__restrict__ coef, const uint8_t *__restrict__ planes,
                               int mode, TurboDst<K> out) {
    turbo_reconstruct<NC, S, SX, SY, K>(frames, coef, planes, mode, out);
}

// grid (output columns / 64, tile rows, frames), block 64 x 8: pixel (x, y) of the frame's clip rectangle, x from the frame's first
// tile column tx0 (tiles of kGenericTileBlocks blocks), y from its first block row ty0. mode (OutMode, uniform over the launch):
// Coded stores the frame's components, Luma the L formula of three, Replicate one sample to three components. kDraft (drafted
// frames, turbo_generic_draft_kernel): plane pitch FrameRecon::idct[c] bw[c], csx / csy the ratios after the reduced IDCT,
// FrameRecon::fancy. CMYK (turbo_cmyk_kernel, turbo_cmyk_draft_kernel: an 8-bit Adobe CMYK or YCCK frame, DESIGN §18): MODE is
// OutMode::CmykRgb or CmykLuma, fixed at compile time like the component count 4 (a run-time count puts v in local memory); the
// four samples go through cmyk_to_rgb (FrameRecon::ycck), and three components or L leave
template <int K, bool kDraft, int MODE = (int)OutMode::Coded>
__device__ __forceinline__ void turbo_generic(const FrameRecon *__restrict__ frames, const uint8_t *__restrict__ planes, int mode, TurboDst<K> out) {
    static_assert(kClipKind<K> && (kBaseKind<K> == kStoreStrided || kBaseKind<K> == kStoreStridedF), "described, cropped destinations");
    constexpr bool kCmyk = MODE == (int)OutMode::CmykRgb || MODE == (int)OutMode::CmykLuma;
    constexpr uint32_t kIn = kCmyk ? 4u : 3u;
    const FrameRecon &f = frames[blockIdx.z];
    const int x = (int)(f.tx0 * (8u * kGenericTileBlocks) + blockIdx.x * 64u + threadIdx.x), y = (int)(8u * (f.ty0 + blockIdx.y) + threadIdx.y);
    if (x < (int)f.clip_x0 || x >= (int)f.clip_x1 || y < (int)f.clip_y0 || y >= (int)f.clip_y1) return;
    const uint32_t nc = kCmyk ? 4u : f.ncomp;
    int v[kIn] = {};
#pragma unroll
    for (uint32_t c = 0; c < kIn; c++) {
        if (c >= nc) break;
        const int fx = f.csx[c], fy = f.csy[c];
        const int w = (int)((f.width + fx - 1) / fx), h = (int)((f.height + fy - 1) / fy);
        if constexpr (kDraft) v[c] = turbo_upsampled(planes + f.sample_base[c], f.idct[c] * f.bw[c], fx, fy, w, h, x, y, f.fancy != 0);
        else v[c] = turbo_upsampled(planes + f.sample_base[c], 8u * f.bw[c], fx, fy, w, h, x, y);
    }
    uint32_t no = nc;
    if constexpr (kCmyk) {
        cmyk_to_rgb(v, f.ycck != 0);
        no = 3;
        if (MODE == (int)OutMode::CmykLuma) v[0] = (19595 * v[0] + 38470 * v[1] + 7471 * v[2] + 32768) >> 16, no = 1;
    } else {
        if (nc == 3 && f.ycbcr) turbo_ycc_rgb(v);
        if (mode == (int)OutMode::Luma) v[0] = (19595 * v[0] + 38470 * v[1] + 7471 * v[2] + 32768) >> 16, no = 1;
        if (mode == (int)OutMode::Replicate) v[1] = v[2] = v[0], no = 3;
    }
#pragma unroll
    for (uint32_t c = 0; c < 3; c++) {
        if (c >= no) break;
        if constexpr (kFloatKind<K>)
            store_elem(out.type, plane_at(out.planes + 4u * f.status_idx + c, x, y), map_int(table_of<kTableKind<K>>(out), c, v[c], pick4(out.scale, c), pick4(out.bias, c)));
        else
            *plane_at(out + 4u * f.status_idx + c, x, y) = (uint8_t)v[c];
    }
}

template <int K>
__global__ void __launch_bounds__(512)
turbo_generic_kernel(const FrameRecon *__restrict__ frames, const uint8_t *__restrict__ planes, int mode, TurboDst<K> out) {
    turbo_generic<K, false>(frames, planes, mode, out);
}

template <int K>
__global__ void __launch_bounds__(512)
turbo_generic_draft_kernel(const FrameRecon *__restrict__ frames, const uint8_t *__restrict__ planes, int mode, TurboDst<K> out) {
    turbo_generic<K, true>(frames, planes, mode, out);
}

// the generic kernels of a CMYK / YCCK group (DESIGN §18), MODE = OutMode::CmykRgb or CmykLuma
template <int K, int MODE>
__global__ void __launch_bounds__(512)
turbo_cmyk_kernel(const FrameRecon *__restrict__ frames, const uint8_t *__restrict__ planes, TurboDst<K> out) {
    turbo_generic<K, false, MODE>(frames, planes, MODE, out);
}

template <int K, int MODE>
__global__ void __launch_bounds__(512)
turbo_cmyk_draft_kernel(const FrameRecon *__restrict__ frames, const uint8_t *__restrict__ planes, TurboDst<K> out) {
    turbo_generic<K, true, MODE>(frames, planes, MODE, out);
}

template <int K, bool kDraft, int MODE>
static void launch_cmyk(const ReconLaunch &l, dim3 grid, TurboDst<K> out, cudaStream_t s) {
    if constexpr (kDraft) turbo_cmyk_draft_kernel<K, MODE><<<grid, dim3(64, 8), 0, s>>>(l.frames, l.planes8, out);
    else turbo_cmyk_kernel<K, MODE><<<grid, dim3(64, 8), 0, s>>>(l.frames, l.planes8, out);
}

// a TurboGeneric group's reconstruction, after its IDCT: the CMYK instances for the modes of four-component frames (DESIGN §18),
// turbo_generic_kernel / turbo_generic_draft_kernel for every other group
template <int K, bool kDraft>
static void launch_c(const ReconLaunch &l, dim3 grid, TurboDst<K> out, cudaStream_t s) {
    if (l.mode == OutMode::CmykRgb) launch_cmyk<K, kDraft, (int)OutMode::CmykRgb>(l, grid, out, s);
    else if (l.mode == OutMode::CmykLuma) launch_cmyk<K, kDraft, (int)OutMode::CmykLuma>(l, grid, out, s);
    else if constexpr (kDraft) turbo_generic_draft_kernel<K><<<grid, dim3(64, 8), 0, s>>>(l.frames, l.planes8, (int)l.mode, out);
    else turbo_generic_kernel<K><<<grid, dim3(64, 8), 0, s>>>(l.frames, l.planes8, (int)l.mode, out);
}

template <int NC, int SX, int SY, int K>
static void launch_b(const ReconLaunch &l, dim3 grid, TurboDst<K> out, cudaStream_t s) {
    turbo_reconstruct_kernel<NC, SX, SY, K><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, l.planes8, (int)l.mode, out);
}

// a drafted Turbo group: grey, or three components whose chroma ratios after the IDCT are 1 x 1 (4:4:4, 4:2:0), 2 x 1 (4:2:2) or
// 1 x 2 (4:4:0) (turbo_path)
template <int S, int K>
static void launch_b_draft(const ReconLaunch &l, dim3 grid, TurboDst<K> out, cudaStream_t s) {
    if (l.ncomp == 1) turbo_reconstruct_draft_kernel<1, S, 1, 1, K><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, l.planes8, (int)l.mode, out);
    else if (l.subx == 2) turbo_reconstruct_draft_kernel<3, S, 2, 1, K><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, l.planes8, (int)l.mode, out);
    else if (l.suby == 2) turbo_reconstruct_draft_kernel<3, S, 1, 2, K><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, l.planes8, (int)l.mode, out);
    else turbo_reconstruct_draft_kernel<3, S, 1, 1, K><<<grid, kThreadsB, 0, s>>>(l.frames, l.coef, l.planes8, (int)l.mode, out);
}

}  // namespace

template <int K>
int launch_turbo(const ReconLaunch &l, void *stream, int *launches) {
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t cblocks = (l.max_bwc * l.max_bhc + kThreadsB - 1) / kThreadsB;
    TurboDst<K> out;
    if constexpr (kFloatKind<K>) {
        out.planes = l.planes;
        out.type = l.convert->type;
        for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++) out.scale[c] = l.convert->scale[c], out.bias[c] = l.convert->bias[c];
        out.table = l.table;
    } else {
        out = l.planes;
    }
    int n = 0;
    if (l.path == ReconPath::Turbo && l.downscale > 1) {  // drafted (DESIGN §17): the luma block is S = 8 / k samples wide
        if (l.ncomp > 1) turbo_idct_draft_kernel<true><<<dim3(cblocks, l.n_frames, l.ncomp - 1), kThreadsB, 0, s>>>(l.frames, l.coef, l.planes8), n++;
        const dim3 grid((l.max_bw0 + kTurboTileW - 1) / kTurboTileW, (l.max_bh0 + kTurboTileH - 1) / kTurboTileH, l.n_frames);
        if (l.downscale == 2) launch_b_draft<4, K>(l, grid, out, s);
        else if (l.downscale == 4) launch_b_draft<2, K>(l, grid, out, s);
        else launch_b_draft<1, K>(l, grid, out, s);
    } else if (l.path == ReconPath::Turbo) {  // the chroma blocks under the clip tiles (FrameRecon::cb_*), then the tiles
        if (l.ncomp > 1) turbo_idct_kernel<true><<<dim3(cblocks, l.n_frames, l.ncomp - 1), kThreadsB, 0, s>>>(l.frames, l.coef, l.planes8), n++;
        const dim3 grid((l.max_bw0 + kTurboTileW - 1) / kTurboTileW, (l.max_bh0 + kTurboTileH - 1) / kTurboTileH, l.n_frames);
        if (l.ncomp == 1) launch_b<1, 1, 1, K>(l, grid, out, s);
        else if (l.subx == 2 && l.suby == 2) launch_b<3, 2, 2, K>(l, grid, out, s);
        else if (l.subx == 2) launch_b<3, 2, 1, K>(l, grid, out, s);
        else if (l.suby == 2) launch_b<3, 1, 2, K>(l, grid, out, s);
        else launch_b<3, 1, 1, K>(l, grid, out, s);
    } else {
        const dim3 grid((8u * l.max_bw0 + 63u) / 64u, l.max_bh0, l.n_frames);
        if (l.downscale > 1) {  // drafted frames (DESIGN §17)
            turbo_idct_draft_kernel<false><<<dim3(cblocks, l.n_frames, l.ncomp), kThreadsB, 0, s>>>(l.frames, l.coef, l.planes8), n++;
            launch_c<K, true>(l, grid, out, s);
        } else {
            turbo_idct_kernel<false><<<dim3(cblocks, l.n_frames, l.ncomp), kThreadsB, 0, s>>>(l.frames, l.coef, l.planes8), n++;
            launch_c<K, false>(l, grid, out, s);
        }
    }
    if (launches) *launches = n + 1;
    return (int)cudaGetLastError();
}

template int launch_turbo<kStoreStrided | kStoreClip>(const ReconLaunch &, void *, int *);
template int launch_turbo<kStoreStridedF | kStoreClip>(const ReconLaunch &, void *, int *);
template int launch_turbo<kStoreStridedF | kStoreClip | kStoreTable>(const ReconLaunch &, void *, int *);

}  // namespace b200jpg
