// resample_sm100.cu -- the resize stage of b200jpg_batch_create_resize (DESIGN §13) and b200jpg_batch_create_resample (DESIGN
// §19): Pillow's Image.reduce and convolution resampler on the reconstruction's uint8 output, every channel on its own, in the
// integer arithmetic of Pillow's 8-bit paths.
//
//   reduce_kernel: grid (row band, frame). Each thread takes output pixels x channels of R along x and sums its fx x fy block of C
//     (fewer pixels in the partial blocks at C's right and bottom edges), so a warp reads each of the fy source rows contiguously.
//     Frames that do not reduce return at once; the kernel is launched only when some frame of the batch reduces.
//   resample_h_kernel: grid (row band, frame). A CTA takes kResampleRows rows of the intermediate (rows y0.. of C); each row of C
//     comes into shared memory with 16-byte loads, and every thread computes output columns x channels from it. The frame's
//     horizontal table is read from shared memory where it fits, otherwise from global memory through L1. A frame whose width does
//     Pillow does not resample horizontally has no horizontal pass: the vertical pass reads the source in the scratch directly.
//   resample_v_kernel: one thread per output pixel, all channels. The taps go down a column of the intermediate, so a warp's loads
//     are contiguous along x and the tap's coefficient is one broadcast load; the clamped sample leaves through the caller's
//     b200jpg_plane descriptor (any signed strides), converted by the float map of b200jpg_batch_decode_into_ex where one is given.
//   resample_v_rgb_kernel: the same for the grey frames of B200JPG_FLAG_OUTPUT_RGB (DESIGN §14), which come last in the frame list:
//     one channel, each value stored to three destinations.
//   cv_resample_h_kernel / cv_resample_v_kernel / cv_area_block_kernel: OpenCV's cv2.resize, INTER_LINEAR and INTER_AREA (DESIGN
//     §20), for batches whose filter is B200JPG_RESAMPLE_CV_*: the same grids, an int32 / float intermediate, blocks summed per
//     output pixel where both axes shrink by integer factors.
// Which passes run is the descriptor's `pass` (Pillow's need_horizontal / need_vertical); a window only selects the tables' rows.
// The host half: resample_coefficients and cv_resample_coefficients, the only places the tables are built (the batch's planning and the test entry
// points b200jpg_resample_coefficients / _box call it). build.py compiles this file with -ffp-contract=off: the double-precision
// arithmetic is evaluated as written, one rounding per operation, on every host.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "internal.hpp"
#include "store_sm90.cuh"

namespace b200jpg {

namespace {

constexpr int kPrecisionBits = 22;  // Pillow's PRECISION_BITS for 8-bit images: 32 - 8 - 2

double box_filter(double x) { return (x > -0.5 && x <= 0.5) ? 1.0 : 0.0; }
double bilinear_filter(double x) {
    if (x < 0.0) x = -x;
    return x < 1.0 ? 1.0 - x : 0.0;
}
double hamming_filter(double x) {
    if (x < 0.0) x = -x;
    if (x == 0.0) return 1.0;
    if (x >= 1.0) return 0.0;
    x = x * M_PI;
    return sin(x) / x * (0.54 + 0.46 * cos(x));
}
double bicubic_filter(double x) {  // Keys, a = -0.5
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
    return 0.0;
}
double sinc_filter(double x) {
    if (x == 0.0) return 1.0;
    x = x * M_PI;
    return sin(x) / x;
}
double lanczos_filter(double x) { return (-3.0 <= x && x < 3.0) ? sinc_filter(x) * sinc_filter(x / 3) : 0.0; }

__device__ __forceinline__ int clamp8(int acc) {
    const int v = acc >> kPrecisionBits;
    return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// Image.reduce's rounding (Pillow's Reduce.c): ((sum + n / 2) * floor(2^24 / n)) >> 24 for a block of n pixels, in uint32 -- the
// product is at most (255 n + n / 2) floor(2^24 / n) <= 255.5 * 2^24 < 2^32. The planning keeps n below 2^24 (fx * fy < 2^24).
__global__ void __launch_bounds__(256) reduce_kernel(const ResampleFrame *__restrict__ frames, uint8_t *__restrict__ scratch) {
    const ResampleFrame &f = frames[blockIdx.y];
    const uint32_t fx = f.fx, fy = f.fy;
    if (fx == 1 && fy == 1) return;
    const uint32_t r0 = blockIdx.x * kReduceRows;
    if (r0 >= f.h) return;
    const uint32_t r1 = min(f.h, r0 + kReduceRows), nc = f.ncomp, outs = f.w * nc;
    for (uint32_t r = r0; r < r1; r++) {
        const uint32_t cy = r * fy, ny = min(fy, f.c_h - cy);
        const uint8_t *rows = scratch + f.c_src + (uint64_t)cy * f.c_pitch;
        uint8_t *o = scratch + f.src + (uint64_t)r * f.src_pitch;
        for (uint32_t k = threadIdx.x; k < outs; k += 256) {
            const uint32_t x = k / nc, c = k - x * nc, cx = x * fx, nx = min(fx, f.c_w - cx);
            const uint8_t *p = rows + (uint64_t)cx * nc + c;
            uint32_t sum = 0;
            for (uint32_t yy = 0; yy < ny; yy++, p += f.c_pitch)
                for (uint32_t xx = 0; xx < nx; xx++) sum += p[xx * nc];
            const uint32_t n = nx * ny;
            o[k] = (uint8_t)(((sum + n / 2) * ((1u << 24) / n)) >> 24);
        }
    }
}

__global__ void __launch_bounds__(256) resample_h_kernel(const ResampleFrame *__restrict__ frames, const uint8_t *__restrict__ input,
                                                         const uint8_t *__restrict__ scratch, uint8_t *__restrict__ inter) {
    extern __shared__ uint4 smem[];
    const ResampleFrame &f = frames[blockIdx.y];
    if (!(f.pass & kPassH)) return;
    const uint32_t rows = f.y1 - f.y0, r0 = blockIdx.x * kResampleRows;
    if (r0 >= rows) return;
    const uint32_t r1 = min(rows, r0 + kResampleRows), nc = f.ncomp, outs = f.tw * nc, ksize = f.h_ksize;
    uint8_t *row_s = reinterpret_cast<uint8_t *>(smem);
    int32_t *coef_s = reinterpret_cast<int32_t *>(row_s + kResampleRowSmem);
    const int32_t *bounds = reinterpret_cast<const int32_t *>(input + f.h_bounds);
    const int32_t *coef = reinterpret_cast<const int32_t *>(input + f.h_coef);
    const bool row_staged = (f.stage & kStageRow) != 0;
    if (f.stage & kStageCoef) {  // (the table is padded to 16 bytes in the input buffer)
        const uint32_t n16 = ((uint32_t)f.tw * ksize + 3) / 4;
        for (uint32_t k = threadIdx.x; k < n16; k += 256) reinterpret_cast<uint4 *>(coef_s)[k] = __ldg(reinterpret_cast<const uint4 *>(coef) + k);
        coef = coef_s;
    }
    __syncthreads();
    for (uint32_t r = r0; r < r1; r++) {
        const uint8_t *src = scratch + f.src + (uint64_t)(f.y0 + r) * f.src_pitch;
        if (row_staged) {  // a scratch row is 16-byte aligned and padded to 16 bytes
            for (uint32_t k = threadIdx.x; k < f.src_pitch / 16; k += 256)
                reinterpret_cast<uint4 *>(row_s)[k] = __ldg(reinterpret_cast<const uint4 *>(src) + k);
            __syncthreads();
            src = row_s;
        }
        uint8_t *o = inter + f.inter + (uint64_t)r * outs;
        for (uint32_t k = threadIdx.x; k < outs; k += 256) {
            const uint32_t x = k / nc, c = k - x * nc;
            const int xmin = __ldg(bounds + 2 * x), n = __ldg(bounds + 2 * x + 1);
            const int32_t *kk = coef + (uint64_t)x * ksize;
            const uint8_t *s = src + (uint32_t)xmin * nc + c;
            int acc = 1 << (kPrecisionBits - 1);
            for (int t = 0; t < n; t++) acc += kk[t] * (int)s[(uint32_t)t * nc];
            o[k] = (uint8_t)clamp8(acc);
        }
        if (row_staged) __syncthreads();  // the row buffer is rewritten for the next row
    }
}

template <bool kFloat, bool kTable = false>
__global__ void __launch_bounds__(256) resample_v_kernel(const ResampleFrame *__restrict__ frames, const uint8_t *__restrict__ input,
                                                         const uint8_t *__restrict__ scratch, const uint8_t *__restrict__ inter, FloatDst out) {
    const ResampleFrame &f = frames[blockIdx.y];
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= (uint64_t)f.tw * f.th) return;
    const uint32_t y = (uint32_t)(i / f.tw), x = (uint32_t)(i - (uint64_t)y * f.tw), nc = f.ncomp;
    const bool hpass = (f.pass & kPassH) != 0;
    const uint8_t *src = hpass ? inter + f.inter : scratch + f.src;  // row 0 of src is row y0 of the source
    const uint64_t pitch = hpass ? (uint64_t)f.tw * nc : f.src_pitch;
    int acc[B200JPG_MAX_COMPONENTS];
    if (f.pass & kPassV) {
        const int32_t *vb = reinterpret_cast<const int32_t *>(input + f.v_bounds);
        const int32_t *kk = reinterpret_cast<const int32_t *>(input + f.v_coef) + (uint64_t)y * f.v_ksize;
        const int n = __ldg(vb + 2 * y + 1);
        const uint8_t *col = src + (uint64_t)(__ldg(vb + 2 * y) - (int)f.y0) * pitch + (uint64_t)x * nc;
#pragma unroll
        for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++) acc[c] = 1 << (kPrecisionBits - 1);
        for (int t = 0; t < n; t++) {
            const int k = __ldg(kk + t);
            const uint8_t *p = col + (uint64_t)t * pitch;
#pragma unroll
            for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++)
                if (c < (int)nc) acc[c] += k * (int)__ldg(p + c);
        }
#pragma unroll
        for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++) acc[c] = clamp8(acc[c]);
    } else {
        const uint8_t *p = src + (uint64_t)y * pitch + (uint64_t)x * nc;
#pragma unroll
        for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++) acc[c] = c < (int)nc ? (int)__ldg(p + c) : 0;
    }
#pragma unroll
    for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++) {
        if (c >= (int)nc) break;
        uint8_t *o = plane_at(out.planes + 4u * f.plane + c, (int)x, (int)y);
        if constexpr (kFloat) store_elem(out.type, o, map_int(table_of<kTable>(out), c, acc[c], pick4(out.scale, c), pick4(out.bias, c)));
        else *o = (uint8_t)acc[c];
    }
}

// resample_v_kernel for the grey frames of B200JPG_FLAG_OUTPUT_RGB: one channel in the scratch and the intermediate, each resampled
// value stored through the frame's three destinations, each with its own component's map
template <bool kFloat, bool kTable = false>
__global__ void __launch_bounds__(256) resample_v_rgb_kernel(const ResampleFrame *__restrict__ frames, const uint8_t *__restrict__ input,
                                                             const uint8_t *__restrict__ scratch, const uint8_t *__restrict__ inter, FloatDst out) {
    const ResampleFrame &f = frames[blockIdx.y];
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= (uint64_t)f.tw * f.th) return;
    const uint32_t y = (uint32_t)(i / f.tw), x = (uint32_t)(i - (uint64_t)y * f.tw);
    const bool hpass = (f.pass & kPassH) != 0;
    const uint8_t *src = hpass ? inter + f.inter : scratch + f.src;  // row 0 of src is row y0 of the source
    const uint64_t pitch = hpass ? (uint64_t)f.tw : f.src_pitch;
    int v;
    if (f.pass & kPassV) {
        const int32_t *vb = reinterpret_cast<const int32_t *>(input + f.v_bounds);
        const int32_t *kk = reinterpret_cast<const int32_t *>(input + f.v_coef) + (uint64_t)y * f.v_ksize;
        const int n = __ldg(vb + 2 * y + 1);
        const uint8_t *col = src + (uint64_t)(__ldg(vb + 2 * y) - (int)f.y0) * pitch + x;
        int acc = 1 << (kPrecisionBits - 1);
        for (int t = 0; t < n; t++) acc += __ldg(kk + t) * (int)__ldg(col + (uint64_t)t * pitch);
        v = clamp8(acc);
    } else {
        v = __ldg(src + (uint64_t)y * pitch + x);
    }
#pragma unroll
    for (int c = 0; c < 3; c++) {
        uint8_t *o = plane_at(out.planes + 4u * f.plane + c, (int)x, (int)y);
        if constexpr (kFloat) store_elem(out.type, o, map_int(table_of<kTable>(out), c, v, out.scale[c], out.bias[c]));
        else *o = (uint8_t)v;
    }
}

// ---- OpenCV's cv2.resize (DESIGN §20): frames with kPassH | kPassV run the two passes of rules 1, 3 and 4 through an intermediate
// of 4 bytes per sample (int32 for the linear rules, float for rule 3); frames with no pass bit sum fx x fy blocks (rule 2, and the
// copy as 1 x 1 blocks). Float arithmetic is one rounding per operation in OpenCV's order (__fmul_rn / __fadd_rn, no contraction).

template <bool kArea>
__global__ void __launch_bounds__(256) cv_resample_h_kernel(const ResampleFrame *__restrict__ frames, const uint8_t *__restrict__ input,
                                                            const uint8_t *__restrict__ scratch, uint8_t *__restrict__ inter) {
    extern __shared__ uint4 smem[];
    const ResampleFrame &f = frames[blockIdx.y];
    if (!(f.pass & kPassH) || ((f.pass & kPassArea) != 0) != kArea) return;
    const uint32_t rows = f.y1 - f.y0, r0 = blockIdx.x * kResampleRows;
    if (r0 >= rows) return;
    const uint32_t r1 = min(rows, r0 + kResampleRows), nc = f.ncomp, outs = f.tw * nc, ksize = f.h_ksize;
    uint8_t *row_s = reinterpret_cast<uint8_t *>(smem);
    int32_t *coef_s = reinterpret_cast<int32_t *>(row_s + kResampleRowSmem);
    const int32_t *bounds = reinterpret_cast<const int32_t *>(input + f.h_bounds);
    const int32_t *coef = reinterpret_cast<const int32_t *>(input + f.h_coef);
    const bool row_staged = (f.stage & kStageRow) != 0;
    if (f.stage & kStageCoef) {
        const uint32_t n16 = ((uint32_t)f.tw * ksize + 3) / 4;
        for (uint32_t k = threadIdx.x; k < n16; k += 256) reinterpret_cast<uint4 *>(coef_s)[k] = __ldg(reinterpret_cast<const uint4 *>(coef) + k);
        coef = coef_s;
    }
    __syncthreads();
    for (uint32_t r = r0; r < r1; r++) {
        const uint8_t *src = scratch + f.src + (uint64_t)(f.y0 + r) * f.src_pitch;
        if (row_staged) {
            for (uint32_t k = threadIdx.x; k < f.src_pitch / 16; k += 256)
                reinterpret_cast<uint4 *>(row_s)[k] = __ldg(reinterpret_cast<const uint4 *>(src) + k);
            __syncthreads();
            src = row_s;
        }
        int32_t *o = reinterpret_cast<int32_t *>(inter + f.inter) + (uint64_t)r * outs;
        for (uint32_t k = threadIdx.x; k < outs; k += 256) {
            const uint32_t x = k / nc, c = k - x * nc;
            const int32_t *kk = coef + (uint64_t)x * ksize;
            if constexpr (kArea) {  // buf[d] = 0; buf[d] += S * alpha, in table order
                const int xmin = __ldg(bounds + 2 * x), n = __ldg(bounds + 2 * x + 1);
                const uint8_t *s = src + (uint32_t)xmin * nc + c;
                float acc = 0.0f;
                for (int t = 0; t < n; t++) acc = __fadd_rn(acc, __fmul_rn((float)s[(uint32_t)t * nc], __int_as_float(kk[t])));
                o[k] = __float_as_int(acc);
            } else {  // S[i0] a0 + S[i1] a1 in int32, no rounding
                const uint32_t i0 = __ldg(bounds + 2 * x), i1 = __ldg(bounds + 2 * x + 1);
                o[k] = (int)src[i0 * nc + c] * kk[0] + (int)src[i1 * nc + c] * kk[1];
            }
        }
        if (row_staged) __syncthreads();
    }
}

__device__ __forceinline__ int clamp255(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// the value of output (x, y), channel c, stored through the frame's destinations: three for the grey frames of
// B200JPG_FLAG_OUTPUT_RGB (kRgb), each with its own component's map
template <bool kFloat, bool kRgb, bool kTable>
__device__ __forceinline__ void cv_store(const ResampleFrame &f, const FloatDst &out, uint32_t x, uint32_t y, int c, int v) {
#pragma unroll
    for (int k = 0; k < (kRgb ? 3 : 1); k++) {
        const int oc = kRgb ? k : c;
        uint8_t *o = plane_at(out.planes + 4u * f.plane + oc, (int)x, (int)y);
        if constexpr (kFloat) store_elem(out.type, o, map_int(table_of<kTable>(out), oc, v, pick4(out.scale, oc), pick4(out.bias, oc)));
        else *o = (uint8_t)v;
    }
}

// one thread per output pixel, all channels; the taps go down a column of the intermediate (rows y0 .. y1 - 1 of the source)
template <bool kArea, bool kFloat, bool kRgb, bool kTable = false>
__global__ void __launch_bounds__(256) cv_resample_v_kernel(const ResampleFrame *__restrict__ frames, const uint8_t *__restrict__ input,
                                                            const uint8_t *__restrict__ inter, FloatDst out) {
    const ResampleFrame &f = frames[blockIdx.y];
    if (!(f.pass & kPassV) || ((f.pass & kPassArea) != 0) != kArea) return;
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= (uint64_t)f.tw * f.th) return;
    const uint32_t y = (uint32_t)(i / f.tw), x = (uint32_t)(i - (uint64_t)y * f.tw), nc = kRgb ? 1u : f.ncomp;
    const uint64_t pitch = (uint64_t)f.tw * nc;  // samples
    const int32_t *vb = reinterpret_cast<const int32_t *>(input + f.v_bounds);
    const int32_t *kk = reinterpret_cast<const int32_t *>(input + f.v_coef) + (uint64_t)y * f.v_ksize;
    const int32_t *T = reinterpret_cast<const int32_t *>(inter + f.inter) + (uint64_t)x * nc;
    if constexpr (kArea) {  // sum = beta0 buf0, then sum += beta_k buf_k; rint, clamp
        const int n = __ldg(vb + 2 * y + 1);
        const int32_t *col = T + (uint64_t)__ldg(vb + 2 * y) * pitch;
        float acc[B200JPG_MAX_COMPONENTS];
#pragma unroll
        for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++) acc[c] = 0.0f;
        for (int t = 0; t < n; t++) {
            const float beta = __int_as_float(__ldg(kk + t));
            const int32_t *p = col + (uint64_t)t * pitch;
#pragma unroll
            for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++)
                if (c < (int)nc) acc[c] = __fadd_rn(acc[c], __fmul_rn(beta, __int_as_float(__ldg(p + c))));
        }
#pragma unroll
        for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++)
            if (c < (int)nc) cv_store<kFloat, kRgb, kTable>(f, out, x, y, c, clamp255(__float2int_rn(acc[c])));
    } else {  // (((b0 (T0 >> 4)) >> 16) + ((b1 (T1 >> 4)) >> 16) + 2) >> 2, clamped
        const int32_t *t0 = T + (uint64_t)__ldg(vb + 2 * y) * pitch, *t1 = T + (uint64_t)__ldg(vb + 2 * y + 1) * pitch;
        const int b0 = __ldg(kk), b1 = __ldg(kk + 1);
#pragma unroll
        for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++)
            if (c < (int)nc)
                cv_store<kFloat, kRgb, kTable>(f, out, x, y, c, clamp255((((b0 * (__ldg(t0 + c) >> 4)) >> 16) + ((b1 * (__ldg(t1 + c) >> 4)) >> 16) + 2) >> 2));
    }
}

// rule 2: output (x, y) is the fx x fy block of the (trimmed) C at (x fx, y fy): (s + 2) >> 2 for 2 x 2 blocks, else
// rint((float)s * (1.0f / (fx fy))); 1 x 1 blocks copy. The planning keeps 255 fx fy below 2^31.
template <bool kFloat, bool kRgb, bool kTable = false>
__global__ void __launch_bounds__(256) cv_area_block_kernel(const ResampleFrame *__restrict__ frames, const uint8_t *__restrict__ scratch,
                                                            FloatDst out) {
    const ResampleFrame &f = frames[blockIdx.y];
    if (f.pass) return;
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= (uint64_t)f.tw * f.th) return;
    const uint32_t y = (uint32_t)(i / f.tw), x = (uint32_t)(i - (uint64_t)y * f.tw), nc = kRgb ? 1u : f.ncomp;
    const uint32_t fx = f.fx, fy = f.fy;
    const uint8_t *p = scratch + f.src + (uint64_t)y * fy * f.src_pitch + (uint64_t)x * fx * nc;
    int s[B200JPG_MAX_COMPONENTS];
#pragma unroll
    for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++) s[c] = 0;
    for (uint32_t yy = 0; yy < fy; yy++, p += f.src_pitch)
        for (uint32_t xx = 0; xx < fx; xx++) {
#pragma unroll
            for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++)
                if (c < (int)nc) s[c] += __ldg(p + xx * nc + c);
        }
    const bool half = fx == 2 && fy == 2;
    const float inv = __fdiv_rn(1.0f, (float)(fx * fy));
#pragma unroll
    for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++)
        if (c < (int)nc) cv_store<kFloat, kRgb, kTable>(f, out, x, y, c, half ? (s[c] + 2) >> 2 : clamp255(__float2int_rn(__fmul_rn((float)s[c], inv))));
}

template <bool kFloat, bool kRgb, bool kTable = false>
void launch_cv_v(const ResampleLaunch &l, const ResampleFrame *frames, uint32_t n, uint32_t gv, const FloatDst &d, cudaStream_t s, int &launches) {
    if (l.cv_kinds & kCvLinear) {
        cv_resample_v_kernel<false, kFloat, kRgb, kTable><<<dim3(gv, n), 256, 0, s>>>(frames, l.input, l.inter, d);
        launches++;
    }
    if (l.cv_kinds & kCvArea) {
        cv_resample_v_kernel<true, kFloat, kRgb, kTable><<<dim3(gv, n), 256, 0, s>>>(frames, l.input, l.inter, d);
        launches++;
    }
    if (l.cv_kinds & kCvBlocks) {
        cv_area_block_kernel<kFloat, kRgb, kTable><<<dim3(gv, n), 256, 0, s>>>(frames, l.scratch, d);
        launches++;
    }
}

}  // namespace

// OpenCV's tables of one axis (DESIGN §20, the encoding of b200jpg_resample_coefficients): inv = (double)out / in, scale = 1 / inv.
// Rules 1 / 4: fx = (float)((d + 0.5) scale - 0.5), sx = floor(fx), fx -= sx (rule 4: sx = floor(d scale), fx = (float)((d + 1) -
// (sx + 1) inv), 0 if <= 0, else its fraction); horizontally fx = 0 and sx clamped at the edges; weights rint((1 - fx) 2048),
// rint(fx 2048) in float. Rule 3: computeResizeAreaTab in double, the weights stored as float.
int cv_resample_coefficients(uint32_t in_size, uint32_t out_size, int table, std::vector<int32_t> &bounds, std::vector<int32_t> &coef,
                             uint32_t &ksize) {
    const int base = table & ~(B200JPG_CV_TABLE_VERTICAL | B200JPG_CV_TABLE_LINEAR);
    if ((base != B200JPG_RESAMPLE_CV_LINEAR && base != B200JPG_RESAMPLE_CV_AREA) || in_size == 0 || out_size == 0)
        return B200JPG_ERR_INVALID_PARAMETER;
    const double inv = (double)out_size / in_size, scale = 1.0 / inv;
    const bool area = base == B200JPG_RESAMPLE_CV_AREA;
    if (area && in_size >= out_size && !(table & B200JPG_CV_TABLE_LINEAR)) {  // rule 3
        std::vector<std::vector<float>> w(out_size);
        bounds.assign(2 * (size_t)out_size, 0);
        ksize = 1;
        for (uint32_t d = 0; d < out_size; d++) {
            const double fsx1 = d * scale, fsx2 = fsx1 + scale, cell = std::min(scale, in_size - fsx1);
            int64_t sx1 = (int64_t)std::ceil(fsx1), sx2 = (int64_t)std::floor(fsx2);
            sx2 = std::min<int64_t>(sx2, (int64_t)in_size - 1);
            sx1 = std::min(sx1, sx2);
            int64_t first = sx1;
            if (sx1 - fsx1 > 1e-3) first = sx1 - 1, w[d].push_back((float)((sx1 - fsx1) / cell));
            for (int64_t sx = sx1; sx < sx2; sx++) w[d].push_back((float)(1.0 / cell));
            if (fsx2 - sx2 > 1e-3) w[d].push_back((float)(std::min(std::min(fsx2 - sx2, 1.0), cell) / cell));
            bounds[2 * (size_t)d] = (int32_t)first;
            bounds[2 * (size_t)d + 1] = (int32_t)w[d].size();
            ksize = std::max<uint32_t>(ksize, (uint32_t)w[d].size());
        }
        coef.assign((size_t)out_size * ksize, 0);
        for (uint32_t d = 0; d < out_size; d++) memcpy(&coef[(size_t)d * ksize], w[d].data(), w[d].size() * sizeof(float));
        return B200JPG_OK;
    }
    const bool vertical = (table & B200JPG_CV_TABLE_VERTICAL) != 0;
    ksize = 2;
    bounds.assign(2 * (size_t)out_size, 0);
    coef.assign(2 * (size_t)out_size, 0);
    const int64_t last = (int64_t)in_size - 1;
    for (uint32_t d = 0; d < out_size; d++) {
        float fx;
        int64_t sx;
        if (!area) {
            fx = (float)((d + 0.5) * scale - 0.5);
            sx = (int64_t)std::floor(fx);
            fx -= (float)sx;
        } else {
            sx = (int64_t)std::floor(d * scale);
            fx = (float)((d + 1) - (sx + 1) * inv);
            fx = fx <= 0 ? 0.0f : fx - (float)std::floor(fx);
        }
        if (!vertical && sx < 0) fx = 0, sx = 0;
        if (!vertical && sx >= last) fx = 0, sx = last;
        bounds[2 * (size_t)d] = (int32_t)std::min(std::max<int64_t>(sx, 0), last);
        bounds[2 * (size_t)d + 1] = (int32_t)std::min(std::max<int64_t>(sx + 1, 0), last);
        coef[2 * (size_t)d] = (int32_t)std::lrint((1.0f - fx) * 2048.0f);
        coef[2 * (size_t)d + 1] = (int32_t)std::lrint(fx * 2048.0f);
    }
    return B200JPG_OK;
}

// Pillow's precompute_coeffs: scale = (double)(in1 - in0) / out_size with the difference taken in float, center = in0 + (j + 0.5)
// scale in double; without a box, scale = in_size / out_size and center = (j + 0.5) scale (DESIGN §13, for any in_size).
int resample_coefficients(uint32_t in_size, const float *box, uint32_t out_size, int resample, std::vector<int32_t> &bounds,
                          std::vector<int32_t> &coef, uint32_t &ksize) {
    double (*filter)(double);
    double s;
    switch (resample) {
    case B200JPG_RESAMPLE_BOX: filter = box_filter, s = 0.5; break;
    case B200JPG_RESAMPLE_BILINEAR: filter = bilinear_filter, s = 1.0; break;
    case B200JPG_RESAMPLE_HAMMING: filter = hamming_filter, s = 1.0; break;
    case B200JPG_RESAMPLE_BICUBIC: filter = bicubic_filter, s = 2.0; break;
    case B200JPG_RESAMPLE_LANCZOS: filter = lanczos_filter, s = 3.0; break;
    default: return B200JPG_ERR_INVALID_PARAMETER;
    }
    if (in_size == 0 || out_size == 0) return B200JPG_ERR_INVALID_PARAMETER;
    const double extent = box ? (double)(box[1] - box[0]) : (double)in_size, in0 = box ? (double)box[0] : 0.0;
    const double scale = extent / out_size, fs = std::max(scale, 1.0), support = s * fs;
    ksize = (uint32_t)ceil(support) * 2 + 1;
    bounds.assign(2 * (size_t)out_size, 0);
    coef.assign((size_t)out_size * ksize, 0);
    std::vector<double> w(ksize);
    for (uint32_t j = 0; j < out_size; j++) {
        const double center = box ? in0 + (j + 0.5) * scale : (j + 0.5) * scale;
        const int64_t xmin = std::max<int64_t>((int64_t)(center - support + 0.5), 0);
        const int64_t n = std::min<int64_t>((int64_t)(center + support + 0.5), in_size) - xmin;
        double ww = 0.0;
        for (int64_t t = 0; t < n; t++) {
            w[t] = filter((t + xmin - center + 0.5) / fs);
            ww += w[t];
        }
        for (int64_t t = 0; t < n; t++) {
            const double v = ww != 0.0 ? w[t] / ww : w[t];
            coef[(size_t)j * ksize + t] = (int32_t)(v < 0 ? -0.5 + v * (1 << kPrecisionBits) : 0.5 + v * (1 << kPrecisionBits));
        }
        bounds[2 * (size_t)j] = (int32_t)xmin;
        bounds[2 * (size_t)j + 1] = (int32_t)n;
    }
    return B200JPG_OK;
}

int launch_resample(const ResampleLaunch &l, void *stream, int *launches) {
    cudaStream_t s = (cudaStream_t)stream;
    int n = 1;
    if (l.resample == B200JPG_RESAMPLE_CV_LINEAR || l.resample == B200JPG_RESAMPLE_CV_AREA) {
        n = 0;
        const uint32_t gh = std::max<uint32_t>(1u, (l.max_rows + kResampleRows - 1) / kResampleRows);
        const uint32_t smem = kResampleRowSmem + kResampleCoefSmem;
        if (l.cv_kinds & kCvLinear) {
            cv_resample_h_kernel<false><<<dim3(gh, l.n_frames), 256, smem, s>>>(l.frames, l.input, l.scratch, l.inter);
            n++;
        }
        if (l.cv_kinds & kCvArea) {
            cv_resample_h_kernel<true><<<dim3(gh, l.n_frames), 256, smem, s>>>(l.frames, l.input, l.scratch, l.inter);
            n++;
        }
        const uint32_t gv = (uint32_t)std::max<uint64_t>(1u, (l.max_pixels + 255) / 256);
        FloatDst d{};
        d.planes = l.planes;
        if (l.convert) {
            d.type = l.convert->type;
            for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++) d.scale[c] = l.convert->scale[c], d.bias[c] = l.convert->bias[c];
            d.table = l.table;
        }
        const uint32_t n_rgb = l.n_frames - l.n_plain;
        if (l.n_plain) {
            if (l.table) launch_cv_v<true, false, true>(l, l.frames, l.n_plain, gv, d, s, n);
            else if (l.convert) launch_cv_v<true, false>(l, l.frames, l.n_plain, gv, d, s, n);
            else launch_cv_v<false, false>(l, l.frames, l.n_plain, gv, d, s, n);
        }
        if (n_rgb) {
            if (l.table) launch_cv_v<true, true, true>(l, l.frames + l.n_plain, n_rgb, gv, d, s, n);
            else if (l.convert) launch_cv_v<true, true>(l, l.frames + l.n_plain, n_rgb, gv, d, s, n);
            else launch_cv_v<false, true>(l, l.frames + l.n_plain, n_rgb, gv, d, s, n);
        }
        if (launches) *launches = n;
        return (int)cudaGetLastError();
    }
    if (l.max_reduce_rows) {
        reduce_kernel<<<dim3((l.max_reduce_rows + kReduceRows - 1) / kReduceRows, l.n_frames), 256, 0, s>>>(l.frames, l.scratch);
        n++;
    }
    const uint32_t gh = std::max<uint32_t>(1u, (l.max_rows + kResampleRows - 1) / kResampleRows);
    resample_h_kernel<<<dim3(gh, l.n_frames), 256, kResampleRowSmem + kResampleCoefSmem, s>>>(l.frames, l.input, l.scratch, l.inter);
    const uint32_t gv = (uint32_t)std::max<uint64_t>(1u, (l.max_pixels + 255) / 256);
    FloatDst d{};
    d.planes = l.planes;
    if (l.convert) {
        d.type = l.convert->type;
        for (int c = 0; c < B200JPG_MAX_COMPONENTS; c++) d.scale[c] = l.convert->scale[c], d.bias[c] = l.convert->bias[c];
        d.table = l.table;
    }
    const uint32_t n_rgb = l.n_frames - l.n_plain;
    if (l.n_plain) {
        if (l.table) resample_v_kernel<true, true><<<dim3(gv, l.n_plain), 256, 0, s>>>(l.frames, l.input, l.scratch, l.inter, d);
        else if (l.convert) resample_v_kernel<true><<<dim3(gv, l.n_plain), 256, 0, s>>>(l.frames, l.input, l.scratch, l.inter, d);
        else resample_v_kernel<false><<<dim3(gv, l.n_plain), 256, 0, s>>>(l.frames, l.input, l.scratch, l.inter, d);
        n++;
    }
    if (n_rgb) {
        const ResampleFrame *rgb = l.frames + l.n_plain;
        if (l.table) resample_v_rgb_kernel<true, true><<<dim3(gv, n_rgb), 256, 0, s>>>(rgb, l.input, l.scratch, l.inter, d);
        else if (l.convert) resample_v_rgb_kernel<true><<<dim3(gv, n_rgb), 256, 0, s>>>(rgb, l.input, l.scratch, l.inter, d);
        else resample_v_rgb_kernel<false><<<dim3(gv, n_rgb), 256, 0, s>>>(rgb, l.input, l.scratch, l.inter, d);
        n++;
    }
    if (launches) *launches = n;
    return (int)cudaGetLastError();
}

}  // namespace b200jpg
