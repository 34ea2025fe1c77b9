// device_layout_client.cpp -- a client of the thorfdbg/libjpeg interface whose BitMapHook hands out one CUDA DEVICE bitmap per
// component, in layouts other than the interleaved canvas: the request carries JPGTAG_B200_DEVICE_BITMAPS. 8-row stripes from
// the top like cmd/reconstruct.cpp:312-342. Every bitmap is pre-filled with 0x5A and holds round8(height) rows, so the rows below
// the image (and the padding columns of the planar layouts) must keep the sentinel.
//   usage: device_layout_client MODE in.jpg out.raw
//     planar    one plane per component, pitch (width + 3) samples
//     bgr       one interleaved canvas, component c at sample depth - 1 - c
//     bottomup  one plane per component, rows from the bottom (negative BytesPerRow), pitch (width + 3) samples
//     planes    JPGTAG_DECODER_UPSAMPLE = false: each component at its own size, requested one by one, planar as above
// 12-bit frames are requested as CTYP_UWORD. out.raw: every component's bitmap as allocated (bgr: the one canvas), in order.
// stdout: "width height depth sample_bytes ok=<0|1> err=<code>", then one line "w rows pitch" per bitmap.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "interface/hooks.hpp"
#include "interface/jpeg.hpp"
#include "interface/parameters.hpp"
#include "interface/tagitem.hpp"

struct Layout {
    int mode;  // 0 planar, 1 bgr, 2 bottomup, 3 planes
    unsigned depth, ss;
    unsigned w[4], rows[4];
    long pitch[4];  // bytes
    unsigned char *dev[4];
};

static JPG_LONG FileHook(struct JPG_Hook *hook, struct JPG_TagItem *tags) {
    FILE *in = (FILE *)hook->hk_pData;
    if (tags->GetTagData(JPGTAG_FIO_ACTION) == JPGFLAG_ACTION_READ)
        return (JPG_LONG)fread(tags->GetTagPtr(JPGTAG_FIO_BUFFER), 1, (size_t)tags->GetTagData(JPGTAG_FIO_SIZE), in);
    return tags->GetTagData(JPGTAG_FIO_ACTION) == JPGFLAG_ACTION_QUERY ? 0 : -1;
}

static JPG_LONG BitmapHook(struct JPG_Hook *hook, struct JPG_TagItem *tags) {
    Layout *l = (Layout *)hook->hk_pData;
    if (tags->GetTagData(JPGTAG_BIO_ACTION) != JPGFLAG_BIO_REQUEST) return 0;
    const int c = (int)tags->GetTagData(JPGTAG_BIO_COMPONENT);
    unsigned char *mem;
    long bpr, bpp;
    if (l->mode == 1) {
        mem = l->dev[0] + (l->depth - 1 - c) * l->ss;
        bpp = (long)(l->depth * l->ss);
        bpr = l->pitch[0];
    } else if (l->mode == 2) {
        mem = l->dev[c] + (l->rows[c] - 1) * l->pitch[c];
        bpp = l->ss;
        bpr = -l->pitch[c];
    } else {
        mem = l->dev[c];
        bpp = l->ss;
        bpr = l->pitch[c];
    }
    tags->SetTagPtr(JPGTAG_BIO_MEMORY, mem);  // a DEVICE pointer
    tags->SetTagData(JPGTAG_BIO_BYTESPERROW, bpr);
    tags->SetTagData(JPGTAG_BIO_BYTESPERPIXEL, bpp);
    tags->SetTagData(JPGTAG_BIO_WIDTH, l->w[l->mode == 1 ? 0 : c]);
    tags->SetTagData(JPGTAG_BIO_HEIGHT, l->rows[l->mode == 1 ? 0 : c]);
    tags->SetTagData(JPGTAG_BIO_PIXELTYPE, l->ss == 2 ? CTYP_UWORD : CTYP_UBYTE);
    return 0;
}

int main(int argc, char **argv) {
    if (argc < 4) return 2;
    Layout l;
    memset(&l, 0, sizeof(l));
    const char *modes[] = {"planar", "bgr", "bottomup", "planes"};
    l.mode = -1;
    for (int m = 0; m < 4; m++)
        if (!strcmp(argv[1], modes[m])) l.mode = m;
    if (l.mode < 0) return 2;
    FILE *in = fopen(argv[2], "rb");
    if (!in) return 2;
    struct JPG_Hook fhook(FileHook, in);
    class JPEG *jpeg = JPEG::Construct(NULL);
    if (!jpeg) return 3;
    struct JPG_TagItem rtags[] = {JPG_PointerTag(JPGTAG_HOOK_IOHOOK, &fhook), JPG_PointerTag(JPGTAG_HOOK_IOSTREAM, in), JPG_EndTag};
    if (!jpeg->Read(rtags)) return 4;
    unsigned char subx[4] = {1, 1, 1, 1}, suby[4] = {1, 1, 1, 1};
    struct JPG_TagItem itags[] = {JPG_ValueTag(JPGTAG_IMAGE_WIDTH, 0), JPG_ValueTag(JPGTAG_IMAGE_HEIGHT, 0), JPG_ValueTag(JPGTAG_IMAGE_DEPTH, 0),
                                  JPG_ValueTag(JPGTAG_IMAGE_PRECISION, 0), JPG_PointerTag(JPGTAG_IMAGE_SUBX, subx),
                                  JPG_PointerTag(JPGTAG_IMAGE_SUBY, suby), JPG_ValueTag(JPGTAG_IMAGE_SUBLENGTH, 4), JPG_EndTag};
    if (!jpeg->GetInformation(itags)) return 5;
    const unsigned width = (unsigned)itags->GetTagData(JPGTAG_IMAGE_WIDTH), height = (unsigned)itags->GetTagData(JPGTAG_IMAGE_HEIGHT);
    l.depth = (unsigned)itags->GetTagData(JPGTAG_IMAGE_DEPTH);
    l.ss = itags->GetTagData(JPGTAG_IMAGE_PRECISION) > 8 ? 2 : 1;
    const unsigned nbuf = l.mode == 1 ? 1 : l.depth;
    for (unsigned c = 0; c < nbuf; c++) {
        const unsigned w = l.mode == 3 ? (width + subx[c] - 1) / subx[c] : width, h = l.mode == 3 ? (height + suby[c] - 1) / suby[c] : height;
        l.w[c] = w;
        l.rows[c] = (h + 7) & ~7u;
        l.pitch[c] = (long)(l.mode == 1 ? w * l.depth : w + 3) * l.ss;
        const size_t bytes = (size_t)l.pitch[c] * l.rows[c];
        if (cudaMalloc((void **)&l.dev[c], bytes) != cudaSuccess || cudaMemset(l.dev[c], 0x5A, bytes) != cudaSuccess) return 6;
    }
    struct JPG_Hook bhook(BitmapHook, &l);
    int ok = 1;
    for (unsigned c = 0; c < (l.mode == 3 ? l.depth : 1u) && ok; c++) {
        for (unsigned y = 0; y < height && ok; y += 8) {
            struct JPG_TagItem dtags[] = {JPG_PointerTag(JPGTAG_BIH_HOOK, &bhook), JPG_ValueTag(JPGTAG_DECODER_MINY, (JPG_LONG)y),
                                          JPG_ValueTag(JPGTAG_DECODER_MAXY, (JPG_LONG)(y + 7 < height ? y + 7 : height - 1)),
                                          JPG_ValueTag(JPGTAG_B200_DEVICE_BITMAPS, 1),
                                          JPG_ValueTag(l.mode == 3 ? JPGTAG_DECODER_UPSAMPLE : JPGTAG_TAG_IGNORE, 0),
                                          JPG_ValueTag(l.mode == 3 ? JPGTAG_DECODER_MINCOMPONENT : JPGTAG_TAG_IGNORE, (JPG_LONG)c),
                                          JPG_ValueTag(l.mode == 3 ? JPGTAG_DECODER_MAXCOMPONENT : JPGTAG_TAG_IGNORE, (JPG_LONG)c), JPG_EndTag};
            ok = jpeg->DisplayRectangle(dtags) != 0;
        }
    }
    const char *e = 0;
    const long code = ok ? 0 : (long)jpeg->LastError(e);
    FILE *out = fopen(argv[3], "wb");
    if (!out) return 2;
    printf("%u %u %u %u ok=%d err=%ld\n", width, height, l.depth, l.ss, ok, code);
    for (unsigned c = 0; c < nbuf; c++) {
        const size_t bytes = (size_t)l.pitch[c] * l.rows[c];
        unsigned char *host = (unsigned char *)malloc(bytes);
        if (!host || cudaMemcpy(host, l.dev[c], bytes, cudaMemcpyDeviceToHost) != cudaSuccess) return 7;
        fwrite(host, 1, bytes, out);
        free(host);
        cudaFree(l.dev[c]);
        printf("%u %u %ld\n", l.w[c], l.rows[c], l.pitch[c]);
    }
    fclose(out);
    JPEG::Destruct(jpeg);
    fclose(in);
    return 0;
}
