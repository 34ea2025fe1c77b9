// jpeg.hpp -- the library object of the JPEG interface (reference: interface/jpeg.hpp:79-250).
//
// Same public surface as the reference's `class JPEG`, so a client written against thorfdbg/libjpeg compiles
// unchanged; behind it sits the GPU decode path (include/b200jpg.h).  Supported here: decoding of baseline /
// extended-sequential Huffman codestreams (Construct, Read, GetInformation, DisplayRectangle, LastError,
// LastWarning, Destruct).  The encoder entry points and the marker peek/read/skip calls exist for link
// compatibility and fail with JPGERR_NOT_IMPLEMENTED.
//
// Deviations from the reference, all on the permissive side (SURVEY.md 8b):
//   * DisplayRectangle is random access and idempotent (the reference is a forward-only stream of 8-row stripes;
//     on that access pattern both produce identical pixels).
//   * Read always consumes the whole codestream; JPGTAG_DECODER_STOP flags are accepted and treated as "run to the
//     end of the image".
#ifndef B200JPG_INTERFACE_JPEG_HPP
#define B200JPG_INTERFACE_JPEG_HPP

#include "jpgtypes.hpp"

struct JPG_TagItem;

class JPG_EXPORT JPEG {
    struct Impl;
    Impl *m_pImpl;
    JPEG(void);
    JPEG(const JPEG &);
    const JPEG &operator=(const JPEG &);
    ~JPEG(void);

public:
    // Optional tags: JPGTAG_B200_DEVICE (CUDA device ordinal). Returns NULL when out of memory.
    static class JPEG *Construct(struct JPG_TagItem *);
    static void Destruct(class JPEG *);

    // Tags: JPGTAG_HOOK_IOHOOK (mandatory), JPGTAG_HOOK_IOSTREAM, JPGTAG_HOOK_BUFFERSIZE, JPGTAG_HOOK_BUFFER.
    JPG_LONG Read(struct JPG_TagItem *);
    JPG_LONG Write(struct JPG_TagItem *);
    // Tags: JPGTAG_BIH_HOOK, JPGTAG_BIO_* defaults, JPGTAG_DECODER_MINX/MINY/MAXX/MAXY/MINCOMPONENT/MAXCOMPONENT,
    // JPGTAG_DECODER_UPSAMPLE, JPGTAG_MATRIX_LTRAFO.
    JPG_LONG DisplayRectangle(struct JPG_TagItem *);
    JPG_LONG ProvideImage(struct JPG_TagItem *);
    // Fills JPGTAG_IMAGE_WIDTH/HEIGHT/DEPTH/PRECISION, the SUBX/SUBY arrays, IS_FLOAT, OUTPUT_CONVERSION.
    JPG_LONG GetInformation(struct JPG_TagItem *);
    JPG_LONG PeekMarker(struct JPG_TagItem *);
    JPG_LONG ReadMarker(void *buffer, JPG_LONG bufsize, struct JPG_TagItem *);
    JPG_LONG SkipMarker(JPG_LONG bytes, struct JPG_TagItem *);
    JPG_LONG WriteMarker(void *buffer, JPG_LONG bufsize, struct JPG_TagItem *);
    // Code of the last failure (0 if none) and its message.
    JPG_LONG LastError(const char *&error);
    JPG_LONG LastWarning(const char *&warning);
};

#endif
