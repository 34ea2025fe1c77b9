// bitmap_sm100.cu -- JPEG::DisplayRectangle into client bitmaps in device memory (JPGTAG_B200_DEVICE_BITMAPS): one request's
// rectangle from the decoded frame to the ImageBitMaps the client's BitMapHook handed out, any pointer and signed strides per
// component (interface/imagebitmap.hpp:104-109), with the block rules of the host copy loop in jpeg_shim.cpp
// (BlockBitmapRequester's walk over whole 8x8 blocks, ImageBitMap::ExtractBitMap imagebitmap.cpp:78-110).
#include <cuda_runtime.h>

#include "internal.hpp"

namespace b200jpg {
namespace {

// one thread per sample position of the rectangle, every requested component
__global__ void __launch_bounds__(256) bitmap_copy_kernel(const BitmapRequest r, const uint8_t *__restrict__ src) {
    const uint32_t w = (uint32_t)(r.x1 - r.x0 + 1);
    const uint64_t i = (uint64_t)blockIdx.x * 256u + threadIdx.x;
    if (i >= (uint64_t)w * (uint32_t)(r.y1 - r.y0 + 1)) return;
    const int x = r.x0 + (int)(i % w), y = r.y0 + (int)(i / w);
    // origin of the part of x's / y's block inside the rectangle: a block whose origin lies outside a bitmap is not written
    const int xb = (x & ~7) > r.x0 ? (x & ~7) : r.x0, yb = (y & ~7) > r.y0 ? (y & ~7) : r.y0;
    for (int k = 0; k < r.ncomp; k++) {
        const BitmapCopy &c = r.comp[k];
        if (!c.dst || (int64_t)c.width <= xb || (int64_t)c.height <= yb) continue;
        const uint64_t at = c.src_off + (uint64_t)y * c.src_pitch + (uint64_t)x * c.src_step;  // in samples
        uint8_t *d = c.dst + (int64_t)x * c.bytes_per_pixel + (int64_t)y * c.bytes_per_row;
        if (!r.wide_out) {
            *d = src[at];
        } else {  // native-endian 16-bit pixels, written bytewise: the client's strides need not be even
            const uint32_t v = r.deep ? (uint32_t)src[2 * at] | ((uint32_t)src[2 * at + 1] << 8) : (uint32_t)src[at];
            d[0] = (uint8_t)v;
            d[1] = (uint8_t)(v >> 8);
        }
    }
}

}  // namespace

int launch_bitmap_copy(const BitmapRequest &r, const uint8_t *src, void *stream) {
    if (r.x1 < r.x0 || r.y1 < r.y0) return 0;
    const uint64_t n = (uint64_t)(r.x1 - r.x0 + 1) * (uint64_t)(r.y1 - r.y0 + 1);
    bitmap_copy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(r, src);
    return (int)cudaGetLastError();
}

}  // namespace b200jpg
