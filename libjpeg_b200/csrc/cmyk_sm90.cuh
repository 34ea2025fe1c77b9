// cmyk_sm90.cuh -- Pillow's conversion of Adobe CMYK and YCCK samples (DESIGN §15), shared by the kernels of both
// reconstructions that decode such frames under an output mode: generic_reconstruct_kernel (recon_sm100.cu) and the turbo
// path's generic kernel (turbo_sm90.cu, DESIGN §18).
#pragma once

namespace b200jpg {

// OutMode::CmykRgb / CmykLuma (DESIGN §15): the clamped 8-bit samples s[0 .. 4) of a CMYK or YCCK frame, in place, as the RGB that
// Pillow's convert("RGB") gives for the frame it reads as Adobe-inverted CMYK ("CMYK;I"). YCCK: Y = s0, Cb = s1 - 128, Cr = s2 - 128
// through libjpeg's ycck_cmyk_convert tables (arithmetic shifts), whose C = 255 - clamp(R) Pillow inverts back to a = clamp(R);
// CMYK: a = 255 - s. Then Pillow's cmyk2rgb with nk = 255 - (255 - s3) = s3: out = s3 - MULDIV255(a, s3)
__device__ __forceinline__ void cmyk_to_rgb(int (&s)[4], bool ycck) {
    int a[3];
    if (ycck) {
        const int y = s[0], cb = s[1] - 128, cr = s[2] - 128;
        a[0] = y + ((91881 * cr + 32768) >> 16);
        a[1] = y + ((-22554 * cb - 46802 * cr + 32768) >> 16);
        a[2] = y + ((116130 * cb + 32768) >> 16);
        for (int c = 0; c < 3; c++) a[c] = a[c] < 0 ? 0 : (a[c] > 255 ? 255 : a[c]);
    } else {
        for (int c = 0; c < 3; c++) a[c] = 255 - s[c];
    }
    const int k = s[3];
    for (int c = 0; c < 3; c++) {
        const int t = a[c] * k + 128;  // MULDIV255
        s[c] = k - (((t >> 8) + t) >> 8);
    }
}

}  // namespace b200jpg
