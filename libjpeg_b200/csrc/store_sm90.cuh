// store_sm90.cuh -- device helpers shared by the kernels that store samples through caller-described destinations
// (recon_sm100.cu, resample_sm100.cu): the float map of b200jpg_batch_decode_into_ex and the b200jpg_plane addressing.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstdint>

#include "b200jpg.h"

namespace b200jpg {

// ---- float elements. The samples arrive as clamped integers 0 <= v < 2^23: 0x4B000000 | v is the float 2^23 + v, so one
// subtraction makes (float)v exactly -- a LOP3 (or the PRMT that takes the byte out of its packed word) and an FADD on the
// otherwise idle FP32 pipe, where I2F would issue at a fraction of that rate. Then fp32_round(fp32_round(v * s) + b), never
// fused.
__device__ __forceinline__ float convert_bits(uint32_t bits, float s, float b) {
    return __fadd_rn(__fmul_rn(__fsub_rn(__uint_as_float(bits), 8388608.f), s), b);
}
__device__ __forceinline__ float convert_int(int v, float s, float b) { return convert_bits(0x4B000000u | (uint32_t)v, s, b); }
// b200jpg_batch_decode_into_table: entry v of component c of the sample tables t (device, 256 floats per component), through the
// non-coherent path -- the 4 KB stay in L1 for the launch
__device__ __forceinline__ float table_at(const float *t, uint32_t c, uint32_t v) {
    float y;
    asm("ld.global.nc.f32 %0, [%1];" : "=f"(y) : "l"(t + 256u * c + v));
    return y;
}
// the sample tables of a float destination d (FloatDst) in a launch whose kind has them (kTable: kStoreTable), else null, so that
// the lookup is compiled out of the affine instances
template <bool kTable, class D>
__device__ __forceinline__ const float *table_of(const D &d) {
    if constexpr (kTable) return d.table;
    else return nullptr;
}
// the float element of the 8-bit sample v of component c: its table entry when the call has tables, else the map
__device__ __forceinline__ float map_int(const float *t, uint32_t c, int v, float s, float b) {
    return t ? table_at(t, c, (uint32_t)v) : convert_int(v, s, b);
}
// scale[c] / bias[c] of a component index known only at run time (a select chain: the parameter bank is not indexed)
__device__ __forceinline__ float pick4(const float (&a)[B200JPG_MAX_COMPONENTS], uint32_t c) {
    return c == 0 ? a[0] : (c == 1 ? a[1] : (c == 2 ? a[2] : a[3]));
}
// one element at o, rounded to the destination type
__device__ __forceinline__ void store_elem(int type, uint8_t *o, float y) {
    if (type == B200JPG_SAMPLE_F32) *reinterpret_cast<float *>(o) = y;
    else if (type == B200JPG_SAMPLE_F16) *reinterpret_cast<__half *>(o) = __float2half_rn(y);
    else *reinterpret_cast<__nv_bfloat16 *>(o) = __float2bfloat16_rn(y);
}

// the sample (x, y) of a described component, signed 64-bit addressing (ImageBitMap, interface/imagebitmap.hpp:104-109).
// The descriptor is read again at every call (L1 hits): held in registers through the line loop of reconstruct_tile, three of
// them push the 4:2:0 kernel over its 96-register budget.
__device__ __forceinline__ uint8_t *plane_at(const b200jpg_plane *p, int x, int y) {
    uint64_t data, bpr;
    int bpp;
    asm volatile("ld.global.nc.u64 %0, [%1];" : "=l"(data) : "l"(&p->data));
    asm volatile("ld.global.nc.s32 %0, [%1];" : "=r"(bpp) : "l"(&p->bytes_per_pixel));
    asm volatile("ld.global.nc.u64 %0, [%1];" : "=l"(bpr) : "l"(&p->bytes_per_row));
    return reinterpret_cast<uint8_t *>(data + (uint64_t)((int64_t)x * bpp) + (uint64_t)((int64_t)y * (int64_t)bpr));
}

}  // namespace b200jpg
