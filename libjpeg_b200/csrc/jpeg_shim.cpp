// jpeg_shim.cpp -- the reference's C++ interface (`class JPEG`, `JPG_TagItem`) on top of the C ABI.
//
// Restates the client-visible protocol of thorfdbg/libjpeg:
//   JPG_TagItem traversal           interface/tagitem.cpp:63-324
//   JPEG::Construct/Destruct/Read   interface/jpeg.cpp:142-353 (I/O hook protocol: io/iostream.cpp:132-223)
//   JPEG::GetInformation            interface/jpeg.cpp:867-954
//   JPEG::DisplayRectangle          interface/jpeg.cpp:694-722, codestream/rectanglerequest.cpp:62-165,
//                                   interface/bitmaphook.cpp:85-248 (24-entry request / release tag array),
//                                   control/bitmapctrl.cpp:142-160, control/blockbitmaprequester.cpp:1229-1244
//                                   (BIO_HEIGHT >> 3 block rows), interface/imagebitmap.cpp:58-125 (canvas anchoring)
//   JPEG::LastError                 interface/jpeg.cpp:962
// Pixels come from b200jpg_decode_to_host (CUDA), or stay on the device for device bitmaps (b200jpg_decode_to_device_ex +
// the copy kernel of bitmap_sm100.cu); there is no CPU decode in here.
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "b200jpg.h"
#include "internal.hpp"
#include "interface/hooks.hpp"
#include "interface/jpeg.hpp"
#include "interface/parameters.hpp"
#include "interface/tagitem.hpp"

// ---------------------------------------------------------------------------------------------------------
// JPG_TagItem
struct JPG_TagItem *JPG_TagItem::NextTagItem(void) {
    struct JPG_TagItem *t = this;
    if (!t) return 0;
    if (t->ti_Tag & JPGTAG_TAG_USER) t++;  // step over the current user tag first
    for (;;) {
        const JPG_Tag id = t->ti_Tag;
        if (id == JPGTAG_TAG_DONE) return 0;
        if (id == JPGTAG_TAG_MORE) {
            t = (struct JPG_TagItem *)t->ti_Data.ti_pPtr;
            if (!t) return 0;
        } else if (id == JPGTAG_TAG_SKIP) {
            t += 1 + t->ti_Data.ti_lData;
        } else if (id & JPGTAG_TAG_USER) {
            return t;
        } else {
            t++;  // IGNORE and every other system tag
        }
    }
}

struct JPG_TagItem *JPG_TagItem::FindTagItem(JPG_Tag wanted) {
    struct JPG_TagItem *t = this;
    if (!t) return 0;
    for (;;) {
        const JPG_Tag id = t->ti_Tag;
        if (id == JPGTAG_TAG_DONE) return 0;
        if (id == JPGTAG_TAG_MORE) {
            t = (struct JPG_TagItem *)t->ti_Data.ti_pPtr;
            if (!t) return 0;
        } else if (id == JPGTAG_TAG_SKIP) {
            t += 1 + t->ti_Data.ti_lData;
        } else {
            if ((id & JPGTAG_TAG_USER) && id == wanted) return t;
            t++;
        }
    }
}

JPG_LONG JPG_TagItem::GetTagData(JPG_Tag id, JPG_LONG def) const {
    const struct JPG_TagItem *t = FindTagItem(id);
    return t ? t->ti_Data.ti_lData : def;
}
JPG_FLOAT JPG_TagItem::GetTagFloat(JPG_Tag id, JPG_FLOAT def) const {
    const struct JPG_TagItem *t = FindTagItem(id);
    return t ? t->ti_Data.ti_fData : def;
}
JPG_APTR JPG_TagItem::GetTagPtr(JPG_Tag id, JPG_APTR def) const {
    const struct JPG_TagItem *t = FindTagItem(id);
    return t ? t->ti_Data.ti_pPtr : def;
}
void JPG_TagItem::SetTagData(JPG_Tag id, JPG_LONG v) {
    if (struct JPG_TagItem *t = FindTagItem(id)) t->ti_Data.ti_lData = v;
}
void JPG_TagItem::SetTagFloat(JPG_Tag id, JPG_FLOAT v) {
    if (struct JPG_TagItem *t = FindTagItem(id)) t->ti_Data.ti_fData = v;
}
void JPG_TagItem::SetTagPtr(JPG_Tag id, JPG_APTR v) {
    if (struct JPG_TagItem *t = FindTagItem(id)) t->ti_Data.ti_pPtr = v;
}
void JPG_TagItem::SetTagSet(void) { ti_Tag |= JPGTAG_SET; }
void JPG_TagItem::ClearTagSets(void) {
    for (struct JPG_TagItem *t = this; t; t = t->NextTagItem()) {
        if (t->ti_Tag & JPGTAG_SET) t->ti_Tag &= ~JPGTAG_SET;
        else t->ti_Tag = JPGTAG_TAG_IGNORE;
    }
}
JPG_LONG JPG_TagItem::FilterTags(struct JPG_TagItem *target, const struct JPG_TagItem *source, const struct JPG_TagItem *defaults,
                                 const struct JPG_TagItem *drop) {
    JPG_LONG count = 0;
    for (const struct JPG_TagItem *t = source; t; t = t->NextTagItem()) {
        if (t->ti_Tag & JPGTAG_TAG_USER) {
            if (target) *target++ = *t;
            count++;
        }
    }
    for (const struct JPG_TagItem *t = defaults; t; t = t->NextTagItem()) {
        if (!(t->ti_Tag & JPGTAG_TAG_USER)) continue;
        if (drop && drop->FindTagItem(t->ti_Tag)) continue;
        if (source && source->FindTagItem(t->ti_Tag)) continue;
        if (target) *target++ = *t;
        count++;
    }
    if (target) {
        target->ti_Tag = JPGTAG_TAG_DONE;
        target->ti_Data.ti_lData = 0;
    }
    return count + 1;
}
struct JPG_TagItem *JPG_TagItem::TagOn(struct JPG_TagItem *add) {
    for (struct JPG_TagItem *t = this; t;) {
        switch (t->ti_Tag) {
        case JPGTAG_TAG_DONE:
            t->ti_Tag = JPGTAG_TAG_MORE;
            t->ti_Data.ti_pPtr = add;
            return t;
        case JPGTAG_TAG_MORE:
            t = (struct JPG_TagItem *)t->ti_Data.ti_pPtr;
            break;
        case JPGTAG_TAG_SKIP:
            t += 1 + t->ti_Data.ti_lData;
            break;
        default:
            t++;
        }
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// JPEG
namespace {

std::mutex g_ctx_mutex;
b200jpg_ctx *g_ctx[64];

int shared_context(int device, b200jpg_ctx **out, std::string &msg) {
    std::lock_guard<std::mutex> lock(g_ctx_mutex);
    const int slot = (device < 0) ? 63 : (device & 63);
    if (!g_ctx[slot]) {
        int rc = b200jpg_create(device, &g_ctx[slot]);
        if (rc) {
            const char *m = 0;
            b200jpg_last_error(0, &m);
            msg = m ? m : "cannot create a CUDA decode context";
            return rc;
        }
    }
    *out = g_ctx[slot];
    return 0;
}

struct BitmapLayout {  // what the client's bitmap hook hands back (interface/imagebitmap.hpp:103)
    uint8_t *mem;
    JPG_ULONG width, height;
    JPG_LONG bytes_per_row;
    int bytes_per_pixel;
    int pixel_type;
    JPG_APTR userdata;
};

}  // namespace

struct JPEG::Impl {
    int device;
    std::vector<uint8_t> stream;  // the codestream as pulled through the I/O hook
    bool have_image;
    b200jpg_frame_info info;
    // decoded frame, interleaved, info.ncomp bytes per pixel (allocated uninitialised: the decode overwrites every byte)
    std::unique_ptr<uint8_t[]> pixels;
    size_t pixel_bytes;
    bool decoded;
    unsigned decoded_flags;  // request flags the cached pixels were decoded with (colour transformation on / off)
    // the same frame kept on the device for clients whose bitmaps are device memory (JPGTAG_B200_DEVICE_BITMAPS)
    uint8_t *d_pixels;
    b200jpg_ctx *d_ctx;
    unsigned d_flags;
    JPG_LONG err_code;
    std::string err_msg;

    Impl() : device(-1), have_image(false), pixel_bytes(0), decoded(false), decoded_flags(0), d_pixels(0), d_ctx(0), d_flags(0), err_code(0) {
        memset(&info, 0, sizeof(info));
    }
    ~Impl() { drop_device_frame(); }
    void drop_device_frame() {
        if (d_pixels) b200jpg_device_free(d_ctx, d_pixels);
        d_pixels = 0;
    }
    JPG_LONG fail(JPG_LONG code, const std::string &msg) {
        err_code = code;
        err_msg = msg;
        return JPG_FALSE;
    }
};

JPEG::JPEG(void) : m_pImpl(0) {}
JPEG::~JPEG(void) {}

class JPEG *JPEG::Construct(struct JPG_TagItem *tags) {
    JPEG *j = new (std::nothrow) JPEG();
    if (!j) return 0;
    j->m_pImpl = new (std::nothrow) Impl();
    if (!j->m_pImpl) {
        delete j;
        return 0;
    }
    if (tags) j->m_pImpl->device = tags->GetTagData(JPGTAG_B200_DEVICE, -1);
    return j;
}

void JPEG::Destruct(class JPEG *j) {
    if (!j) return;
    delete j->m_pImpl;
    delete j;
}

JPG_LONG JPEG::Read(struct JPG_TagItem *tags) {
    Impl &s = *m_pImpl;
    struct JPG_Hook *hook = tags ? (struct JPG_Hook *)tags->GetTagPtr(JPGTAG_HOOK_IOHOOK) : 0;
    if (!hook) return s.fail(JPGERR_OBJECT_DOESNT_EXIST, "no IOHook defined to read the data from");  // jpeg.cpp:264-266
    if (s.have_image) return JPG_TRUE;  // the whole image was parsed by the first call
    JPG_APTR handle = tags->GetTagPtr(JPGTAG_HOOK_IOSTREAM);
    JPG_LONG bufsize = tags->GetTagData(JPGTAG_HOOK_BUFFERSIZE, 2048);
    if (bufsize <= 0) bufsize = 2048;
    if (bufsize < (1 << 16)) bufsize = 1 << 16;  // fewer hook round trips; any size is legal for the client
    std::vector<uint8_t> buf((size_t)bufsize);
    JPG_APTR userbuf = tags->GetTagPtr(JPGTAG_HOOK_BUFFER);
    s.stream.clear();
    for (;;) {  // io/iostream.cpp:174-189: READ action, the hook may substitute its own buffer
        struct JPG_TagItem io[] = {JPG_PointerTag(JPGTAG_FIO_BUFFER, userbuf ? userbuf : (JPG_APTR)buf.data()),
                                   JPG_ValueTag(JPGTAG_FIO_SIZE, userbuf ? tags->GetTagData(JPGTAG_HOOK_BUFFERSIZE, 2048) : bufsize),
                                   JPG_PointerTag(JPGTAG_FIO_HANDLE, handle),
                                   JPG_ValueTag(JPGTAG_FIO_ACTION, JPGFLAG_ACTION_READ),
                                   JPG_PointerTag(JPGTAG_FIO_USERDATA, hook->hk_pData),
                                   JPG_EndTag};
        JPG_LONG got = hook->CallLong(io);
        if (got < 0) return s.fail(got, "IOHook signalled an error on reading");  // iostream.cpp:185-188
        if (got == 0) break;
        const uint8_t *p = (const uint8_t *)io[0].ti_Data.ti_pPtr;
        s.stream.insert(s.stream.end(), p, p + got);
    }
    if (s.stream.empty()) return s.fail(JPGERR_UNEXPECTED_EOF, "unexpected EOF while parsing the image");
    int rc = b200jpg_parse(s.stream.data(), s.stream.size(), &s.info);
    if (rc) {
        const char *m = 0;
        b200jpg_last_error(0, &m);
        return s.fail(rc, m ? m : "cannot parse the codestream");
    }
    s.have_image = true;
    s.decoded = false;
    s.err_code = 0;
    return JPG_TRUE;
}

JPG_LONG JPEG::GetInformation(struct JPG_TagItem *tags) {
    Impl &s = *m_pImpl;
    if (!s.have_image) return s.fail(JPGERR_OBJECT_DOESNT_EXIST, "no image loaded to request information from");
    if (!tags) return JPG_TRUE;
    tags->SetTagData(JPGTAG_IMAGE_WIDTH, (JPG_LONG)s.info.width);
    tags->SetTagData(JPGTAG_IMAGE_HEIGHT, (JPG_LONG)s.info.height);
    tags->SetTagData(JPGTAG_IMAGE_DEPTH, s.info.ncomp);
    tags->SetTagData(JPGTAG_IMAGE_PRECISION, s.info.precision);
    JPG_ULONG tablesz = (JPG_ULONG)tags->GetTagData(JPGTAG_IMAGE_SUBLENGTH);
    if (tablesz) {  // jpeg.cpp:893-916
        uint8_t *sx = (uint8_t *)tags->GetTagPtr(JPGTAG_IMAGE_SUBX), *sy = (uint8_t *)tags->GetTagPtr(JPGTAG_IMAGE_SUBY);
        if (sx) memset(sx, 0, tablesz);
        if (sy) memset(sy, 0, tablesz);
        for (JPG_ULONG c = 0; c < s.info.ncomp && c < tablesz; c++) {
            if (sx) sx[c] = s.info.subx[c];
            if (sy) sy[c] = s.info.suby[c];
        }
    }
    tags->SetTagData(JPGTAG_IMAGE_IS_FLOAT, 0);           // jpeg.cpp:843-861 without a merging spec box
    tags->SetTagData(JPGTAG_IMAGE_OUTPUT_CONVERSION, 0);
    if (struct JPG_TagItem *t = tags->FindTagItem(JPGTAG_ALPHA_MODE)) t->ti_Tag = JPGTAG_TAG_IGNORE;     // no alpha channel
    if (struct JPG_TagItem *t = tags->FindTagItem(JPGTAG_ALPHA_TAGLIST)) t->ti_Tag = JPGTAG_TAG_IGNORE;  // :944-950
    return JPG_TRUE;
}

JPG_LONG JPEG::DisplayRectangle(struct JPG_TagItem *tags) {
    Impl &s = *m_pImpl;
    if (!s.have_image) return s.fail(JPGERR_OBJECT_DOESNT_EXIST, "no image loaded that could be displayed");
    // ---- BitMapHook defaults + hook (bitmaphook.cpp:85-125)
    BitmapLayout def = {0, 0, 0, 0, 0, 0, 0};
    struct JPG_Hook *hook = 0;
    // ---- rectangle request (rectanglerequest.cpp:62-165)
    JPG_LONG minx = 0, miny = 0, maxx = (JPG_LONG)s.info.width - 1, maxy = (JPG_LONG)s.info.height - 1;
    JPG_LONG firstc = 0, lastc = s.info.ncomp - 1;
    bool upsample = true, colortrafo = true, device_bitmaps = false;
    for (const struct JPG_TagItem *t = tags; t; t = t->NextTagItem()) {
        const JPG_LONG v = t->ti_Data.ti_lData;
        switch (t->ti_Tag) {
        case JPGTAG_BIO_MEMORY: def.mem = (uint8_t *)t->ti_Data.ti_pPtr; break;
        case JPGTAG_BIO_WIDTH: def.width = (JPG_ULONG)v; break;
        case JPGTAG_BIO_HEIGHT: def.height = (JPG_ULONG)v; break;
        case JPGTAG_BIO_BYTESPERROW: def.bytes_per_row = v; break;
        case JPGTAG_BIO_BYTESPERPIXEL: def.bytes_per_pixel = (uint8_t)v; break;
        case JPGTAG_BIO_PIXELTYPE: def.pixel_type = (uint8_t)v; break;
        case JPGTAG_BIO_USERDATA: def.userdata = t->ti_Data.ti_pPtr; break;
        case JPGTAG_BIH_HOOK: hook = (struct JPG_Hook *)t->ti_Data.ti_pPtr; break;
        case JPGTAG_DECODER_MINX:
            if (v < 0) return s.fail(JPGERR_OVERFLOW_PARAMETER, "Rectangle MinX underflow, must be >= 0");
            if (v > minx) minx = v;
            break;
        case JPGTAG_DECODER_MINY:
            if (v < 0) return s.fail(JPGERR_OVERFLOW_PARAMETER, "Rectangle MinY underflow, must be >= 0");
            if (v > miny) miny = v;
            break;
        case JPGTAG_DECODER_MAXX:
            if (v < 0) return s.fail(JPGERR_OVERFLOW_PARAMETER, "Rectangle MaxX underflow, must be >= 0");
            if (v < maxx) maxx = v;
            break;
        case JPGTAG_DECODER_MAXY:
            if (v < 0) return s.fail(JPGERR_OVERFLOW_PARAMETER, "Rectangle MaxY underflow, must be >= 0");
            if (v < maxy) maxy = v;
            break;
        case JPGTAG_DECODER_MINCOMPONENT:
            if (v < 0 || v > 65535) return s.fail(JPGERR_OVERFLOW_PARAMETER, "MinComponent overflow, must be >= 0 && < 65536");
            if (v > firstc) firstc = v;
            break;
        case JPGTAG_DECODER_MAXCOMPONENT:
            if (v < 0 || v > 65535) return s.fail(JPGERR_OVERFLOW_PARAMETER, "MaxComponent overflow, must be >= 0 && < 65536");
            if (v < lastc) lastc = v;
            break;
        case JPGTAG_B200_DEVICE_BITMAPS: device_bitmaps = v != 0; break;
        case JPGTAG_DECODER_UPSAMPLE: upsample = v != 0; break;
        case JPGTAG_MATRIX_LTRAFO: colortrafo = v != JPGFLAG_MATRIX_COLORTRANSFORMATION_NONE; break;
        default: break;
        }
    }
    if (maxx < minx || maxy < miny) return s.fail(JPGERR_INVALID_PARAMETER, "the requested rectangle is empty");
    // without upsampling there is no colour transformation either (rectanglerequest.cpp:155-158), and the components come one
    // per request, each in its own subsampled coordinates (BitmapCtrl::SubsampledRegion, bitmapctrl.cpp:273-293)
    if (!upsample) {
        colortrafo = false;
        if (firstc != lastc)
            return s.fail(JPGERR_INVALID_PARAMETER, "if upsampling is disabled, components can only be reconstructed one by one");
    }
    // a subset of the components: the identity transformation works component by component; through YCbCr->RGB the reference
    // feeds zeros for the components left out (blockbitmaprequester.cpp:1046-1051) -- not offered here
    if ((firstc != 0 || lastc != s.info.ncomp - 1) && colortrafo && s.info.ycbcr)
        return s.fail(JPGERR_NOT_IMPLEMENTED, "a subset of the components through the colour transformation is not supported by the GPU path");
    const int sample_bytes = s.info.precision > 8 ? 2 : 1;
    // planes mode: plane offsets (in samples) and sizes of the components at their own resolution
    size_t plane_at[B200JPG_MAX_COMPONENTS + 1] = {0};
    uint32_t plane_w[B200JPG_MAX_COMPONENTS] = {0};
    for (int c = 0; c < s.info.ncomp; c++) {
        plane_w[c] = (s.info.width + s.info.subx[c] - 1) / s.info.subx[c];
        plane_at[c + 1] = plane_at[c] + (size_t)plane_w[c] * ((s.info.height + s.info.suby[c] - 1) / s.info.suby[c]);
    }
    // the rectangle the samples are copied for: the request's, or its subsampled image (the hook still sees the request's)
    JPG_LONG cminx = minx, cmaxx = maxx, cminy = miny, cmaxy = maxy;
    if (!upsample && firstc <= lastc) {
        const int sx = s.info.subx[firstc], sy = s.info.suby[firstc];
        cminx = (minx + sx - 1) / sx, cmaxx = (maxx + sx) / sx - 1;
        cminy = (miny + sy - 1) / sy, cmaxy = (maxy + sy) / sy - 1;
    }

    // ---- decode on first use (CUDA; the whole frame, kept for later rectangles)
    const unsigned want_flags = !upsample ? (B200JPG_FLAG_NO_UPSAMPLE | B200JPG_FLAG_NO_COLOR_TRANSFORM)
                                          : ((!colortrafo && s.info.ycbcr) ? B200JPG_FLAG_NO_COLOR_TRANSFORM : 0u);
    if (device_bitmaps) {
        if (!s.d_pixels || s.d_flags != want_flags) {
            b200jpg_ctx *ctx = 0;
            std::string msg;
            int rc = shared_context(s.device, &ctx, msg);
            if (rc) return s.fail(rc, msg);
            s.drop_device_frame();
            const uint8_t *frames[1] = {s.stream.data()};
            size_t lens[1] = {s.stream.size()};
            rc = b200jpg_decode_to_device_ex(ctx, frames, lens, 1, want_flags, &s.d_pixels, 0);
            if (rc) {
                const char *m = 0;
                b200jpg_last_error(0, &m);
                return s.fail(rc, (m && *m) ? m : "decoding failed");
            }
            s.d_ctx = ctx;
            s.d_flags = want_flags;
        }
    } else if (!s.decoded || s.decoded_flags != want_flags) {
        b200jpg_ctx *ctx = 0;
        std::string msg;
        int rc = shared_context(s.device, &ctx, msg);
        if (rc) return s.fail(rc, msg);
        s.pixel_bytes = (upsample ? (size_t)s.info.width * s.info.height * s.info.ncomp : plane_at[s.info.ncomp]) * sample_bytes + 256;
        s.pixels.reset(new (std::nothrow) uint8_t[s.pixel_bytes]);
        if (!s.pixels) return s.fail(JPGERR_OUT_OF_MEMORY, "out of memory for the decoded frame");
        const uint8_t *frames[1] = {s.stream.data()};
        size_t lens[1] = {s.stream.size()};
        // JPEG objects decode concurrently: a batch owns its buffers and its stream, the context's buffer pool locks itself
        rc = b200jpg_decode_to_host_ex(ctx, frames, lens, 1, s.pixels.get(), s.pixel_bytes, want_flags);
        if (rc) {
            const char *m = 0;
            b200jpg_last_error(0, &m);  // this thread's failure (the context is shared with other JPEG objects)
            return s.fail(rc, (m && *m) ? m : "decoding failed");
        }
        s.decoded = true;
        s.decoded_flags = want_flags;
    }

    // ---- REQUEST per component (bitmaphook.cpp:130-209), pixel types must agree (bitmapctrl.cpp:152-158)
    const int nc = s.info.ncomp;
    BitmapLayout lay[B200JPG_MAX_COMPONENTS];
    struct JPG_TagItem bt[24];
    auto fill = [&](int action, int comp, const BitmapLayout &l) {
        const int sx = s.info.subx[comp], sy = s.info.suby[comp];
        bt[0] = JPG_ValueTag(JPGTAG_BIO_ACTION, action);
        bt[1] = JPG_PointerTag(JPGTAG_BIO_MEMORY, l.mem);
        bt[2] = JPG_ValueTag(JPGTAG_BIO_WIDTH, l.width);
        bt[3] = JPG_ValueTag(JPGTAG_BIO_HEIGHT, l.height);
        bt[4] = JPG_ValueTag(JPGTAG_BIO_BYTESPERROW, l.bytes_per_row);
        bt[5] = JPG_ValueTag(JPGTAG_BIO_BYTESPERPIXEL, l.bytes_per_pixel);
        bt[6] = JPG_ValueTag(JPGTAG_BIO_PIXELTYPE, action == JPGFLAG_BIO_REQUEST ? def.pixel_type : l.pixel_type);
        bt[7] = JPG_ValueTag(JPGTAG_BIO_ROI, 0);
        bt[8] = JPG_ValueTag(JPGTAG_BIO_COMPONENT, comp);
        bt[9] = JPG_PointerTag(JPGTAG_BIO_USERDATA, l.userdata);
        bt[10] = JPG_ValueTag(JPGTAG_BIO_MINX, minx);
        bt[11] = JPG_ValueTag(JPGTAG_BIO_MINY, miny);
        bt[12] = JPG_ValueTag(JPGTAG_BIO_MAXX, maxx);
        bt[13] = JPG_ValueTag(JPGTAG_BIO_MAXY, maxy);
        bt[14] = JPG_ValueTag(JPGTAG_BIO_ALPHA, 0);
        bt[15] = JPG_ValueTag(JPGTAG_TAG_IGNORE, 0);
        bt[16] = JPG_ValueTag(JPGTAG_TAG_IGNORE, comp);
        bt[17] = JPG_ValueTag(JPGTAG_BIO_PIXEL_MINX, (minx + sx - 1) / sx);
        bt[18] = JPG_ValueTag(JPGTAG_BIO_PIXEL_MINY, (miny + sy - 1) / sy);
        bt[19] = JPG_ValueTag(JPGTAG_BIO_PIXEL_MAXX, (maxx + sx) / sx - 1);
        bt[20] = JPG_ValueTag(JPGTAG_BIO_PIXEL_MAXY, (maxy + sy) / sy - 1);
        bt[21] = JPG_ValueTag(JPGTAG_BIO_PIXEL_XORG, 0);
        bt[22] = JPG_ValueTag(JPGTAG_BIO_PIXEL_YORG, 0);
        bt[23] = JPG_EndTag;
    };
    int common_type = 0;
    JPG_ULONG max_block_row = 0xffffffffu;  // blockbitmaprequester.cpp:1240
    for (int c = (int)firstc; c <= (int)lastc; c++) {
        fill(JPGFLAG_BIO_REQUEST, c, def);
        if (hook) {
            JPG_LONG r = hook->CallLong(bt);
            if (r < 0) return s.fail(r, "BitMapHook signalled an error");
        }
        BitmapLayout &l = lay[c];
        l.mem = (uint8_t *)bt[1].ti_Data.ti_pPtr;
        l.width = (JPG_ULONG)bt[2].ti_Data.ti_lData;
        l.height = (JPG_ULONG)bt[3].ti_Data.ti_lData;
        l.bytes_per_row = bt[4].ti_Data.ti_lData;
        l.bytes_per_pixel = (uint8_t)bt[5].ti_Data.ti_lData;
        l.pixel_type = (uint8_t)bt[6].ti_Data.ti_lData;
        l.userdata = bt[9].ti_Data.ti_pPtr;
        if (common_type == 0) common_type = l.pixel_type;
        else if (l.pixel_type && l.pixel_type != common_type)
            return s.fail(JPGERR_INVALID_PARAMETER, "pixel types must be consistent across components");
        const JPG_ULONG mr = (l.height >> 3) - 1;  // unsigned, wraps for heights below 8 exactly like the reference
        if (mr < max_block_row) max_block_row = mr;
    }
    // colortransformerfactory.cpp:613-632: bytes only hold 8-bit frames; 16-bit samples hold any precision of this path
    const bool deep = s.info.precision > 8;
    if (common_type != 0 && common_type != CTYP_UBYTE && common_type != CTYP_UWORD)
        return s.fail(JPGERR_INVALID_PARAMETER, "only CTYP_UBYTE and CTYP_UWORD pixels are supported by the GPU path");
    if (deep && common_type == CTYP_UBYTE)
        return s.fail(JPGERR_OVERFLOW_PARAMETER, "invalid data type selected for the image, image precision is deeper than 8 bits");
    const bool wide_out = common_type == CTYP_UWORD;

    // ---- copy, block by block like the reference walks the region (PushReconstructedData / ReconstructUnsampled)
    const uint32_t W = s.info.width;
    // the usual client bitmap -- one interleaved canvas, component c at base + c -- is copied run-wise instead of bytewise
    bool interleaved = nc > 1 && upsample && firstc == 0 && lastc == nc - 1;
    for (int c = 0; c < nc && interleaved; c++)
        interleaved = interleaved && deep == wide_out && lay[c].mem && lay[c].pixel_type && lay[c].mem == lay[0].mem + c * (deep ? 2 : 1) &&
                      lay[c].bytes_per_pixel == nc * (deep ? 2 : 1) &&
                      lay[c].bytes_per_row == lay[0].bytes_per_row && lay[c].width == lay[0].width && lay[c].height == lay[0].height;
    // block rows up to min(MaxY >> 3, (smallest BIO_HEIGHT >> 3) - 1) are reconstructed (blockbitmaprequester.cpp:1166-1167)
    long long last_by = (long long)(cmaxy >> 3);
    if ((long long)max_block_row < last_by) last_by = (long long)max_block_row;
    if (device_bitmaps) {
        // the client's bitmaps are device memory: the rectangle goes from the frame kept on the device to every requested
        // component's bitmap in one kernel, with the rules of the loop below (whole blocks whose origin lies outside a bitmap,
        // a NULL base or pixel type 0 leave the component unwritten, imagebitmap.cpp:78-110), any pointer and strides
        b200jpg::BitmapRequest r{};
        r.x0 = (int)cminx, r.x1 = (int)cmaxx, r.y0 = (int)cminy, r.y1 = (int)cmaxy;
        if (last_by * 8 + 7 < (long long)r.y1) r.y1 = (int)(last_by * 8 + 7);
        r.deep = deep, r.wide_out = wide_out;
        for (int c = (int)firstc; c <= (int)lastc; c++) {
            const BitmapLayout &l = lay[c];
            b200jpg::BitmapCopy &k = r.comp[r.ncomp++];
            k.dst = (l.mem && l.pixel_type) ? l.mem : nullptr;
            k.bytes_per_pixel = l.bytes_per_pixel, k.bytes_per_row = l.bytes_per_row;
            k.width = l.width, k.height = l.height;
            // sample (x, y) of component c: in the interleaved frame, or in the component's own plane (as in the loop below)
            k.src_off = upsample ? (uint64_t)c : (uint64_t)plane_at[c];
            k.src_step = upsample ? (uint32_t)nc : 1u;
            k.src_pitch = upsample ? W * (uint32_t)nc : plane_w[c];
        }
        if (r.y1 >= r.y0) {
            int rc = b200jpg::device_bitmap_copy(s.d_ctx, r, s.d_pixels);
            if (rc) {
                const char *m = 0;
                b200jpg_last_error(0, &m);
                return s.fail(rc, (m && *m) ? m : "device bitmap copy failed");
            }
        }
        last_by = -1;  // nothing left for the host loop
    }
    for (long long by = (long long)(cminy >> 3); by <= last_by; by++) {
        const JPG_LONG y0 = (by == (cminy >> 3)) ? cminy : (JPG_LONG)(by << 3);
        const JPG_LONG y1 = ((JPG_LONG)(by << 3) + 7 < cmaxy) ? (JPG_LONG)(by << 3) + 7 : cmaxy;
        for (JPG_LONG bx = cminx >> 3; bx <= (cmaxx >> 3); bx++) {
            const JPG_LONG x0 = (bx == (cminx >> 3)) ? cminx : (bx << 3);
            const JPG_LONG x1 = ((bx << 3) + 7 < cmaxx) ? (bx << 3) + 7 : cmaxx;
            for (int c = (int)firstc; c <= (int)lastc; c++) {
                const BitmapLayout &l = lay[c];
                // ImageBitMap::ExtractBitMap: a block whose origin lies outside the client bitmap, a NULL base
                // or pixel type 0 leave the component unwritten (imagebitmap.cpp:78-110)
                if (!l.mem || !l.pixel_type || l.width <= (JPG_ULONG)x0 || l.height <= (JPG_ULONG)y0) continue;
                for (JPG_LONG y = y0; y <= y1; y++) {
                    // sample (x0, y) of component c: in the interleaved frame, or in the component's own plane
                    const size_t at = upsample ? ((size_t)y * W + (size_t)x0) * nc + c : plane_at[c] + (size_t)y * plane_w[c] + (size_t)x0;
                    const size_t step = upsample ? (size_t)nc : 1;
                    const uint8_t *src = s.pixels.get() + at * sample_bytes;
                    uint8_t *dst = l.mem + (ptrdiff_t)x0 * l.bytes_per_pixel + (ptrdiff_t)y * l.bytes_per_row;
                    if (interleaved) {  // all components of the run in one go (the other components skip this block)
                        if (c == 0) memcpy(dst, src, (size_t)(x1 - x0 + 1) * nc * sample_bytes);
                    } else if (!wide_out) {
                        for (JPG_LONG x = x0; x <= x1; x++, src += step, dst += l.bytes_per_pixel) *dst = *src;
                    } else if (!deep) {  // 8-bit samples into 16-bit pixels
                        for (JPG_LONG x = x0; x <= x1; x++, src += step, dst += l.bytes_per_pixel) {
                            const uint16_t v = *src;
                            memcpy(dst, &v, 2);
                        }
                    } else {
                        for (JPG_LONG x = x0; x <= x1; x++, src += 2 * step, dst += l.bytes_per_pixel) memcpy(dst, src, 2);
                    }
                }
            }
        }
    }
    // ---- RELEASE per component (bitmaphook.cpp:214-248)
    for (int c = (int)firstc; c <= (int)lastc; c++) {
        fill(JPGFLAG_BIO_RELEASE, c, lay[c]);
        if (hook) {
            JPG_LONG r = hook->CallLong(bt);
            if (r < 0) return s.fail(r, "BitMapHook signalled an error");
        }
    }
    return JPG_TRUE;
}

JPG_LONG JPEG::LastError(const char *&error) {
    error = m_pImpl->err_code ? m_pImpl->err_msg.c_str() : 0;
    return m_pImpl->err_code;
}
JPG_LONG JPEG::LastWarning(const char *&warning) {
    warning = 0;
    return 0;
}

// encoder side and marker access: present for link compatibility only
JPG_LONG JPEG::Write(struct JPG_TagItem *) { return m_pImpl->fail(JPGERR_NOT_IMPLEMENTED, "encoding is not part of the GPU decode path"); }
JPG_LONG JPEG::ProvideImage(struct JPG_TagItem *) { return m_pImpl->fail(JPGERR_NOT_IMPLEMENTED, "encoding is not part of the GPU decode path"); }
JPG_LONG JPEG::PeekMarker(struct JPG_TagItem *) {
    m_pImpl->fail(JPGERR_NOT_IMPLEMENTED, "marker access is not part of the GPU decode path");
    return -1;
}
JPG_LONG JPEG::ReadMarker(void *, JPG_LONG, struct JPG_TagItem *) {
    m_pImpl->fail(JPGERR_NOT_IMPLEMENTED, "marker access is not part of the GPU decode path");
    return -1;
}
JPG_LONG JPEG::SkipMarker(JPG_LONG, struct JPG_TagItem *) {
    m_pImpl->fail(JPGERR_NOT_IMPLEMENTED, "marker access is not part of the GPU decode path");
    return -1;
}
JPG_LONG JPEG::WriteMarker(void *, JPG_LONG, struct JPG_TagItem *) {
    m_pImpl->fail(JPGERR_NOT_IMPLEMENTED, "marker access is not part of the GPU decode path");
    return -1;
}
