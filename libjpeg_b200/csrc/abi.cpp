// abi.cpp -- implementation of the C ABI declared in include/b200jpg.h (compiled by nvcc as host C++).
//
// Host side of the decode path: parses the codestreams (parse.cpp), groups scans that share geometry and
// tables into launch classes, lays the batch out in HBM (see internal.hpp) and drives the two CUDA stages.
// There is no CPU decode path in here: without a CUDA device every decode entry point fails.
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>  // header-only NVTX 3: ranges show up in Nsight Systems timelines, cost nothing without a tool attached

#include <algorithm>
#include <array>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <tuple>
#include <type_traits>
#include <vector>

#include "internal.hpp"
#include "specsync.hpp"

namespace {
struct NvtxRange {  // SURVEY 5 (tracing): one range per stage of the path
    explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};
}  // namespace

using namespace b200jpg;

namespace {

thread_local std::string g_tls_error;
thread_local int g_tls_code = 0;

inline uint64_t align_up(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }

}  // namespace

static void set_thread_error(int code, const std::string &msg) {
    g_tls_code = code;
    g_tls_error = msg;
}

// Device / pinned-host buffers are recycled through the context: a streaming caller creates and destroys one batch per
// chunk of frames, and cudaMalloc / cudaHostAlloc per chunk would dominate the host side of the pipeline.
struct PoolBuf {
    void *p;
    size_t bytes;
    int kind;  // 0 = pinned host, 1 = device
};

struct b200jpg_ctx {
    int device = 0;
    std::string error;
    int code = 0;
    std::mutex pool_mutex;
    std::vector<PoolBuf> pool;
    void *get(int kind, size_t bytes, cudaError_t *err) {
        *err = cudaSuccess;
        if (bytes == 0) bytes = 256;
        {
            std::lock_guard<std::mutex> lock(pool_mutex);
            int best = -1;
            for (size_t i = 0; i < pool.size(); i++)
                if (pool[i].kind == kind && pool[i].bytes >= bytes && pool[i].bytes <= bytes + bytes / 2 + (1u << 20) &&
                    (best < 0 || pool[i].bytes < pool[(size_t)best].bytes))
                    best = (int)i;
            if (best >= 0) {
                void *p = pool[(size_t)best].p;
                pool.erase(pool.begin() + best);
                return p;
            }
        }
        void *p = nullptr;
        *err = kind ? cudaMalloc(&p, bytes) : cudaHostAlloc(&p, bytes, cudaHostAllocDefault);
        if (*err != cudaSuccess) {  // make room and retry once
            trim();
            *err = kind ? cudaMalloc(&p, bytes) : cudaHostAlloc(&p, bytes, cudaHostAllocDefault);
        }
        return *err == cudaSuccess ? p : nullptr;
    }
    void put(int kind, void *p, size_t bytes) {
        if (!p) return;
        if (bytes == 0) bytes = 256;
        std::lock_guard<std::mutex> lock(pool_mutex);
        pool.push_back(PoolBuf{p, bytes, kind});
    }
    void trim() {
        std::lock_guard<std::mutex> lock(pool_mutex);
        for (auto &b : pool) {
            if (b.kind) cudaFree(b.p);
            else cudaFreeHost(b.p);
        }
        pool.clear();
    }
    int fail(int c, const std::string &m) {
        {
            std::lock_guard<std::mutex> lock(pool_mutex);  // contexts are shared between threads (the JPEG shim)
            code = c;
            error = m;
        }
        set_thread_error(c, m);  // b200jpg_last_error(NULL, ...) on the failing thread always sees its own failure
        return c;
    }
    int fail_cuda(cudaError_t e, const char *what) {
        return fail(B200JPG_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
    }
};

namespace {

struct ScanClass {
    ScanClassParams p{};
    int table_set = 0;
    std::vector<ClassScan> scans;
    std::vector<uint64_t> interval_off;  // absolute offsets into the packed byte buffer
    std::vector<uint64_t> interval_end;
    std::vector<uint64_t> clean_off;     // offsets into the unstuffed buffer
    std::vector<uint8_t> scan_on_device; // per scan: its restart index is built by restart_index_kernel
    std::vector<uint64_t> scan_ecs_off, scan_ecs_end;  // per scan, absolute
    uint64_t interval_base = 0;          // index of this class's first interval in d_interval_len
    uint64_t spec_base = 0;              // indexed classes: first work item of this class in the spec arrays
    bool fused = false;                  // progressive class decoded by the component-fused kernels (its frames form a PfGroupHost)
    int frame_comp0 = 0;                 // frame component of the scan's first component
    // offsets (bytes) of the device copies inside the input buffer
    uint64_t dev_scans = 0, dev_intervals = 0, dev_interval_end = 0, dev_clean_off = 0;
};

// What the frames of one reconstruction group share: component count, chroma factors and path, and the parts of their plans that
// change the launches or the store kind
struct GroupKey {
    uint32_t ncomp = 0, subx = 1, suby = 1;
    ReconPath path = ReconPath::Tiled;
    int orientation = 1;  // B200JPG_FLAG_EXIF_ORIENTATION: the frames' orientation; 2..8 store through rewritten descriptors
    bool cropped = false; // the frames' tiles cover their rectangles, clipped stores (FrameRecon::clip_*)
    bool resized = false; // cropped frames stored as uint8 into the scratch, never converted
    bool described = false;  // the frames store through rewritten descriptors (FramePlan::described)
    OutMode mode = OutMode::Coded;  // B200JPG_FLAG_OUTPUT_RGB / _L
    uint32_t scale = 1;   // the frames' factor k (ReconLaunch::downscale)
    auto fields() const { return std::tie(ncomp, subx, suby, path, orientation, cropped, resized, described, mode, scale); }
    bool operator==(const GroupKey &o) const { return fields() == o.fields(); }
};

struct ReconGroup {
    GroupKey key;
    std::vector<FrameRecon> frames;
    uint32_t max_bw0 = 0, max_bh0 = 0, max_bwc = 0, max_bhc = 0;
    uint64_t dev_frames = 0;
};

// progressive frames whose scan script lets a component be decoded in one go (progfused_sm100.cu): the classes of its scans
struct PfGroupHost {
    std::vector<int> dc;       // interleaved DC scans, file order
    std::vector<int> ac[4];    // single-component AC scans per frame component, file order
    int comp_of_ac[4] = {0, 0, 0, 0};
};

// scans share a launch class when their launch parameters and their table set are equal, compared bytewise
struct ClassKey {
    ScanClassParams p;
    int table_set;
    bool operator<(const ClassKey &o) const { return memcmp(this, &o, sizeof(ClassKey)) < 0; }
};
static_assert(std::has_unique_object_representations_v<ClassKey>, "ClassKey is compared bytewise: ScanClassParams must have no padding");

struct Extent {
    uint64_t w, h;
};
// the factor k of B200JPG_FLAG_DOWNSCALE_k: 1, 2, 4 or 8
uint32_t downscale_of(unsigned flags) { return 1u << ((flags & B200JPG_FLAG_DOWNSCALE_MASK) >> 2); }
constexpr unsigned kOutputModes = B200JPG_FLAG_OUTPUT_RGB | B200JPG_FLAG_OUTPUT_L;

bool rect_empty(const b200jpg_rect &r) { return r.x == 0 && r.y == 0 && r.width == 0 && r.height == 0; }
bool size_empty(const b200jpg_size &s) { return s.width == 0 && s.height == 0; }
bool box_empty(const b200jpg_box &b) { return b.x0 == 0.0 && b.y0 == 0.0 && b.x1 == 0.0 && b.y1 == 0.0; }
bool resample_known(int r) { return r >= B200JPG_RESAMPLE_LANCZOS && r <= B200JPG_RESAMPLE_HAMMING; }  // PIL's values 1 .. 5
bool resample_cv(int r) { return r == B200JPG_RESAMPLE_CV_LINEAR || r == B200JPG_RESAMPLE_CV_AREA; }  // OpenCV's (DESIGN §20)

// Pillow's draft scale (JpegImageFile.draft) of a frame of codestream size W x H for a request of width x height (both >= 1): the
// largest k of 8, 4, 2, 1 with k <= min(W / width, H / height), 1 when none fits
uint32_t draft_scale_of(const b200jpg_frame_info &fi, uint32_t width, uint32_t height) {
    const uint32_t s = std::min(fi.width / width, fi.height / height);
    for (uint32_t k : {8u, 4u, 2u})
        if (k <= s) return k;
    return 1;
}

// libjpeg-turbo's IDCT output size of component c at scale 1/k (jdmaster.c, DESIGN §17): m = 8 / k, doubled while below 8 and the
// component's ratios to the largest factors stay even multiples
uint32_t draft_idct_size(const b200jpg_frame_info &fi, int c, uint32_t k) {
    uint32_t hmax = 1, vmax = 1;
    for (int j = 0; j < fi.ncomp; j++) hmax = std::max<uint32_t>(hmax, fi.hs[j]), vmax = std::max<uint32_t>(vmax, fi.vs[j]);
    const uint32_t m = 8 / k;
    uint32_t s = m;
    while (s < 8 && (hmax * m) % (fi.hs[c] * s * 2) == 0 && (vmax * m) % (fi.vs[c] * s * 2) == 0) s *= 2;
    return s;
}

// the integer factors component c of a frame decoded at scale 1/k is upsampled by after its IDCT: hmax (8 / k) / (h_c s_c) x
// vmax (8 / k) / (v_c s_c), s_c = draft_idct_size (DESIGN §17); subx x suby at k = 1
struct Ratio {
    uint32_t x, y;
};
Ratio draft_ratio(const b200jpg_frame_info &fi, int c, uint32_t k) {
    uint32_t hmax = 1, vmax = 1;
    for (int j = 0; j < fi.ncomp; j++) hmax = std::max<uint32_t>(hmax, fi.hs[j]), vmax = std::max<uint32_t>(vmax, fi.vs[j]);
    const uint32_t s = draft_idct_size(fi, c, k);
    return {hmax * (8 / k) / (fi.hs[c] * s), vmax * (8 / k) / (fi.vs[c] * s)};
}

// What live frame i of a batch is asked for and how it is decoded (b200jpg_batch::plan), filled once by the planning steps of
// batch_create_impl and read by every later step and both decode calls. A JPEG XT residual codestream's record is its frame's, with
// its own ncomp (parse_residual checks that they agree), so that the two stay in one reconstruction group.
struct FramePlan {
    // frame_plan (B200JPG_FLAG_OUTPUT_RGB / _L, DESIGN §14): the path, the components the reconstruction covers and the components the
    // frame leaves with. Without a mode bit: recon_path and the frame's own components.
    ReconPath path = ReconPath::Tiled;
    uint32_t ncomp = 0;      // components reconstructed, from component 0 on
    uint32_t out_ncomp = 0;  // components written
    OutMode mode = OutMode::Coded;
    uint32_t k = 1;          // decoded at 1/k: B200JPG_FLAG_DOWNSCALE_k, or the frame's draft (admit_drafts)
    int orientation = 1;     // the Exif orientation the frame leaves with: its own with B200JPG_FLAG_EXIF_ORIENTATION, else 1
    // admit_crops: C, a rectangle of the oriented output at 1/k -- the caller's, or the whole output for a resized frame and under
    // B200JPG_FLAG_LIBJPEG_TURBO -- trimmed by plan_resample to the part the resize reads
    bool cropped = false;
    b200jpg_rect crop{};
    // admit_sizes / admit_boxes (DESIGN §19): the target W_t x H_t, Pillow's source box and the window ({0, ..}: the defaults); the
    // frame leaves with the window's extent, or the target's; rs: its index into b200jpg_batch::rs_frames (plan_resample)
    bool resized = false;
    b200jpg_size target{};
    b200jpg_box box{};
    b200jpg_rect window{};
    int rs = -1;
    // the caller's B200JPG_FLIP_H / _V (DESIGN §21). A frame without a size has it folded into `orientation` (frame_plan) and
    // `crop` (admit_crops); a resized frame's resample pass stores through its destinations mirrored over the window
    // (stage_frame_planes): the flip stays behind the resize, with which it does not commute
    uint8_t flip = 0;
    // oriented, cropped (so resized) or written in an output mode: the reconstruction stores through the frame's destinations
    // rewritten into decoded coordinates (rewrite_frame), in place of the packed slot it takes otherwise
    bool described = false;
};

// component c as it leaves the decoder, decoded at scale 1/k: the frame size W' x H' = ceil(W / k) x ceil(H / k), or without
// upsampling its own ceil(W' / subx) x ceil(H' / suby) -- the extent the kernels decode
Extent decoded_extent(const b200jpg_frame_info &fi, int c, unsigned flags, uint64_t k) {
    uint64_t w = (fi.width + k - 1) / k, h = (fi.height + k - 1) / k;
    if (flags & B200JPG_FLAG_NO_UPSAMPLE) w = (w + fi.subx[c] - 1) / fi.subx[c], h = (h + fi.suby[c] - 1) / fi.suby[c];
    return {w, h};
}

// ... and as the frame of plan p leaves: width and height swapped for the Exif orientations 5..8; the size of C for a cropped frame
// (C is given in those output coordinates and checked against them; never together with B200JPG_FLAG_NO_UPSAMPLE); the window's or
// the target's size for a resized one
Extent out_extent(const b200jpg_frame_info &fi, int c, unsigned flags, const FramePlan &p) {
    if (p.resized) return rect_empty(p.window) ? Extent{p.target.width, p.target.height} : Extent{p.window.width, p.window.height};
    if (p.cropped) return {p.crop.width, p.crop.height};
    const Extent e = decoded_extent(fi, c, flags, p.k);
    return p.orientation >= 5 ? Extent{e.h, e.w} : e;
}

// A destination described in output coordinates (data d, pixel stride p, row stride r) as seen from the decoded coordinates
// (x, y) of a component of decoded extent w x h under Exif orientation o (DESIGN §11): the kernels walk (x, y) and store
// through the rewritten descriptor. Returns false when the new pixel stride does not fit its int32 field.
bool orient_plane(b200jpg_plane &pl, int o, uint64_t w, uint64_t h) {
    const int64_t p = pl.bytes_per_pixel, r = pl.bytes_per_row, W = (int64_t)w - 1, H = (int64_t)h - 1;
    int64_t off, np, nr;
    switch (o) {
    case 2: off = W * p, np = -p, nr = r; break;
    case 3: off = W * p + H * r, np = -p, nr = -r; break;
    case 4: off = H * r, np = p, nr = -r; break;
    case 5: off = 0, np = r, nr = p; break;
    case 6: off = H * p, np = r, nr = -p; break;
    case 7: off = H * p + W * r, np = -r, nr = -p; break;
    case 8: off = W * r, np = -r, nr = p; break;
    default: return true;
    }
    if (np < INT32_MIN || np > INT32_MAX) return false;
    pl.data = static_cast<uint8_t *>(pl.data) + off;
    pl.bytes_per_pixel = (int32_t)np;
    pl.bytes_per_row = nr;
    return true;
}

// A destination of a cropped image (the rectangle r of the output) as the destination of the uncropped output: d - x p - y r, in
// 64-bit integer arithmetic on the address. The kernels store only inside the clip rectangle (crop_to_decoded), so nothing is ever
// written through it outside the caller's bitmap.
void translate_plane(b200jpg_plane &pl, const b200jpg_rect &r) {
    const uint64_t a = reinterpret_cast<uintptr_t>(pl.data) - (uint64_t)((int64_t)r.x * pl.bytes_per_pixel) - (uint64_t)((int64_t)r.y * pl.bytes_per_row);
    pl.data = reinterpret_cast<void *>((uintptr_t)a);
}

// [x0, x1) x [y0, y1) in the decoded coordinates the kernels walk
struct Clip {
    uint32_t x0, y0, x1, y1;
};
// The rectangle r of the output image of orientation o as a rectangle of the decoded (downscaled, upright) image of extent w x h:
// the inverse of the mapping orient_plane applies (output (u, v) = decoded (w-1-x, y) for 2, (y, x) for 5, ...)
Clip crop_to_decoded(int o, const b200jpg_rect &r, uint64_t w, uint64_t h) {
    const uint32_t W = (uint32_t)w, H = (uint32_t)h;
    const uint32_t u0 = r.x, u1 = r.x + r.width, v0 = r.y, v1 = r.y + r.height;  // output columns / rows
    switch (o) {
    case 2: return {W - u1, v0, W - u0, v1};
    case 3: return {W - u1, H - v1, W - u0, H - v0};
    case 4: return {u0, H - v1, u1, H - v0};
    case 5: return {v0, u0, v1, u1};
    case 6: return {v0, H - u1, v1, H - u0};
    case 7: return {W - v1, H - u1, W - v0, H - u0};
    case 8: return {W - v1, u0, W - v0, u1};
    default: return {u0, v0, u1, v1};
    }
}

// The orientation that writes F(T_o(D)), for the Exif orientation o (T_o: DESIGN §11) and the flip F (B200JPG_FLIP_H / _V bits,
// DESIGN §21): the dihedral product, kFlipOrientation[o - 1][F]
constexpr uint8_t kFlipOrientation[8][4] = {{1, 2, 4, 3}, {2, 1, 3, 4}, {3, 4, 2, 1}, {4, 3, 1, 2},
                                            {5, 6, 8, 7}, {6, 5, 7, 8}, {7, 8, 6, 5}, {8, 7, 5, 6}};

// The rectangle r of an image of extent w x h as the rectangle of the flipped image that holds the same samples
b200jpg_rect flip_rect(const b200jpg_rect &r, uint32_t flip, uint64_t w, uint64_t h) {
    b200jpg_rect m = r;
    if (flip & B200JPG_FLIP_H) m.x = (uint32_t)(w - r.x - r.width);
    if (flip & B200JPG_FLIP_V) m.y = (uint32_t)(h - r.y - r.height);
    return m;
}

// A destination of a tw x th image made the destination of its flipped image: (x, y) goes where (tw - 1 - x, y) (B200JPG_FLIP_H)
// and (x, th - 1 - y) (B200JPG_FLIP_V) went, as orient_plane mirrors for the orientations 2 and 4
void flip_plane(b200jpg_plane &pl, uint32_t flip, uint64_t tw, uint64_t th) {
    uint64_t a = reinterpret_cast<uintptr_t>(pl.data);
    if (flip & B200JPG_FLIP_H) a += (uint64_t)((int64_t)(tw - 1) * pl.bytes_per_pixel), pl.bytes_per_pixel = -pl.bytes_per_pixel;
    if (flip & B200JPG_FLIP_V) a += (uint64_t)((int64_t)(th - 1) * pl.bytes_per_row), pl.bytes_per_row = -pl.bytes_per_row;
    pl.data = reinterpret_cast<void *>((uintptr_t)a);
}

// body(i) for every frame i < n, on at most max_threads host threads
template <class Body>
void for_frames(int n, unsigned max_threads, const Body &body) {
    const unsigned nt = std::min({std::max(1u, std::thread::hardware_concurrency()), max_threads, (unsigned)n});
    std::vector<std::thread> pool;
    for (unsigned t = 0; t < nt; t++)
        pool.emplace_back([&, t]() {
            for (int i = (int)t; i < n; i += (int)nt) body(i);
        });
    for (auto &th : pool) th.join();
}

}  // namespace

struct b200jpg_batch {
    b200jpg_ctx *ctx = nullptr;
    int n = 0;
    unsigned flags = 0;  // B200JPG_FLAG_*
    std::vector<ParsedFrame> frames;
    std::vector<int> parse_status;
    // [n] every live frame's request and plan (FramePlan): every extent, plane layout, path and store decision of a frame reads it
    // here -- its factor k included (DESIGN §17)
    std::vector<FramePlan> plan;
    int n_user = 0;                      // frames of the caller; [n_user, n) are residual codestreams of JPEG XT frames
    std::vector<int> xt_child, xt_parent;  // [n_user] index of a frame's residual frame or -1; [n] the reverse
    std::vector<uint64_t> out_off, out_bytes;
    uint64_t out_total = 0;
    std::vector<std::array<uint64_t, 4>> coef_base;  // [n] int16 element offset of every component's coefficient plane (live frames)
    std::vector<TableSet> table_sets;
    std::vector<uint64_t> dev_tables;  // offset of each table blob inside the input buffer
    std::vector<ScanClass> classes;
    std::vector<ReconGroup> groups;
    std::vector<IndexScan> index_scans;  // scans whose restart index is built on the device, at upload
    uint64_t dev_index_scans = 0;
    std::vector<PfGroupHost> pf_groups;  // progressive frames decoded component by component
    std::vector<uint16_t> pf_dc_quant;   // per group: quantiser of coefficient 0 per frame component (4 each)
    int16_t *d_dcplane = nullptr;        // fused progressive groups: one DC level per block
    std::vector<ProgFrame> prog_frames;  // progressive frames of the scan-by-scan path: dequantised after their last scan
    uint64_t dev_prog_frames = 0;
    uint32_t prog_max_blocks = 0;
    uint64_t ecs_bytes = 0, stored_blocks = 0;
    bool clear_coef = false;  // some component of some frame is coded by no scan: its plane must read as zeros

    // staging / device memory
    uint8_t *h_input = nullptr;  // pinned
    uint64_t input_bytes = 0;    // codestream bytes + descriptors
    uint64_t bytes_region = 0;   // size of the codestream region at the start of the input buffer
    uint8_t *d_input = nullptr;
    int16_t *d_coef = nullptr;
    uint64_t coef_elems = 0;
    int32_t *d_samples = nullptr;     // int32 planes: exact pass of frames flagged `narrow`
    int16_t *d_samples16 = nullptr;   // int16 planes: every frame
    uint64_t sample_elems = 0;
    uint8_t *d_planes8 = nullptr;     // B200JPG_FLAG_LIBJPEG_TURBO: the uint8 planes of turbo_idct_kernel
    uint64_t plane8_bytes = 0;
    uint8_t *d_clean = nullptr;
    uint64_t clean_bytes = 0;
    uint32_t *d_interval_len = nullptr;
    uint32_t *d_overrun = nullptr;    // per class {count, interval indices}: class ci starts at interval_base + ci
    uint8_t *d_spec = nullptr;        // restart-less scans: segments, exits, entries, counts, DC sums of all indexed classes
    size_t sz_spec = 0;
    uint64_t n_spec = 0;              // work items over all indexed classes
    size_t sz_overrun = 0;
    uint64_t n_intervals = 0;
    uint32_t *d_status = nullptr;
    std::vector<uint32_t> h_status;
    bool status_fetched = false;
    bool uploaded = false;

    size_t sz_status = 0, sz_ilen = 0;
    cudaEvent_t ev_last = nullptr;  // recorded after the last work enqueued for this batch: destroy waits for it
    // b200jpg_batch_decode_into: the descriptor table [4 * n], staged in a ring of kPlaneSlots pinned copies and copied on the
    // call's stream; ev_planes[k] is recorded behind the copy out of slot k, which is rewritten only after it. With several
    // slots the host may run that many calls ahead of the device.
    // Behind the table, 256-byte aligned, each slot has room for the 4 KB of sample tables of b200jpg_batch_decode_into_table, which
    // ride the same copy.
    static constexpr int kPlaneSlots = 3;
    static constexpr uint64_t kTableBytes = sizeof(float) * B200JPG_MAX_COMPONENTS * 256;
    b200jpg_plane *h_planes = nullptr, *d_planes = nullptr;
    cudaEvent_t ev_planes[kPlaneSlots] = {};
    int plane_slot = 0;
    // some live frame is described (FramePlan::described): its group stores through rewritten descriptors
    bool rewritten = false;
    // resized frames: the filter and the reducing_gap (<= 0: None) of the batch; per resized frame its resample descriptor and its
    // tables (h bounds, h coefficients, v bounds, v coefficients). The descriptor table of a decode holds 4 * (n + resized frames)
    // entries: the destinations of resized frame r at 4 * (n + r)
    int resample = 0;
    double gap = 0.0;
    std::vector<ResampleFrame> rs_frames;
    uint32_t rs_plain = 0; // resized frames [rs_plain, ..) are grey frames of B200JPG_FLAG_OUTPUT_RGB (ResampleLaunch::n_plain)
    std::vector<std::array<std::vector<int32_t>, 4>> rs_tables;
    uint64_t dev_rs_frames = 0;
    uint32_t rs_max_rows = 0, rs_max_reduce_rows = 0;
    uint32_t rs_cv_kinds = 0;  // OpenCV's filters: kCvLinear / kCvArea / kCvBlocks of the resized frames (ResampleLaunch::cv_kinds)
    uint64_t rs_max_pixels = 0;
    uint8_t *d_scratch = nullptr, *d_inter = nullptr;  // C of every resized frame; the horizontal pass's rows
    uint64_t scratch_bytes = 0, inter_bytes = 0;
    size_t n_planes() const { return 4 * ((size_t)n + rs_frames.size()); }
    uint64_t table_offset() const { return align_up(sizeof(b200jpg_plane) * n_planes(), 256); }  // of the sample tables in a slot
    uint64_t slot_bytes() const { return table_offset() + kTableBytes; }
    int last_launches = 0;
    bool timing = false;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};  // start, after a0, after a1, after b
};

extern "C" {

// Frames of one source share their tables: the decoder tables of a scan are built once per distinct set of inputs of
// build_table_set -- the scan's Huffman specifications, quantisation tables, point transform and spectral selection -- and copied
// for the other scans that have the same (b200jpg_selftest_table_cache checks the cache against fresh builds on the host).
struct TableCache {
    std::map<std::string, TableSet> built;
};

static std::string table_inputs_key(const ScanInfo &sc) {
    std::string k;
    k.reserve(2048);
    auto put = [&](const void *p, size_t n) { k.append(reinterpret_cast<const char *>(p), n); };
    const int head[6] = {sc.progressive ? 1 : 0, sc.ss, sc.se, sc.ah, sc.lowbit, sc.ns};
    put(head, sizeof(head));
    put(sc.td, sizeof(sc.td));
    put(sc.ta, sizeof(sc.ta));
    for (int pass = 0; pass < 2; pass++)
        for (int t = 0; t < 4; t++) {
            const HuffSpec &h = pass ? sc.ac[t] : sc.dc[t];
            const uint8_t d = h.defined ? 1 : 0;
            put(&d, 1);
            if (!h.defined) continue;
            put(h.bits, 16);
            put(&h.nvals, sizeof(h.nvals));
            put(h.vals, (size_t)std::min(std::max(h.nvals, 0), 256));
        }
    for (int t = 0; t < 4; t++) {
        const uint8_t d = sc.quant_defined[t] ? 1 : 0;
        put(&d, 1);
        if (d) put(sc.quant[t], sizeof(sc.quant[t]));
    }
    return k;
}

static int build_table_set_cached(const ScanInfo &sc, TableSet &out, std::string &err, TableCache &cache) {
    std::string key = table_inputs_key(sc);
    auto it = cache.built.find(key);
    if (it != cache.built.end()) {
        out = it->second;
        return B200JPG_OK;
    }
    const int rc = build_table_set(sc, out, err);
    if (rc == B200JPG_OK) cache.built.emplace(std::move(key), out);
    return rc;
}

// JPEG XT: the residual codestream of `base` (its RESI box) as a frame of its own; what of it the path covers
static int parse_residual(const ParsedFrame &base, ParsedFrame &rf, std::string &err, bool device_index) {
    int rst;
    try {
        rst = parse_codestream(base.xt.resi.data(), base.xt.resi.size(), rf, err, device_index);
    } catch (...) {
        rst = B200JPG_ERR_MALFORMED_STREAM;
        err = "could not be parsed";
    }
    const b200jpg_frame_info &bi = base.info, &ri = rf.info;
    if (rst == 0 && (rf.xt.present || ri.width != bi.width || ri.height != bi.height || ri.ncomp != bi.ncomp || ri.precision != 8)) {
        rst = B200JPG_ERR_NOT_IMPLEMENTED;
        err = "outside the JPEG XT profile of the GPU path (8-bit DCT residual of the frame's size)";
    }
    if (rst != 0) err = "residual codestream: " + err;
    return rst;
}

// b200jpg_parse and b200jpg_exif_orientation: one parse, the residual codestream of a JPEG XT frame included
static int parse_one(const uint8_t *data, size_t len, ParsedFrame &pf) {
    std::string err;
    int rc;
    try {
        rc = parse_codestream(data, len, pf, err);
        if (rc == 0 && pf.xt.present) {
            ParsedFrame rf;
            rc = parse_residual(pf, rf, err, false);
        }
    } catch (const std::bad_alloc &) {
        rc = B200JPG_ERR_OUT_OF_MEMORY;
        err = "out of memory while parsing the codestream";
    }
    g_tls_code = rc;
    g_tls_error = err;
    return rc;
}

int b200jpg_parse(const uint8_t *data, size_t len, b200jpg_frame_info *info) {
    ParsedFrame pf;
    const int rc = parse_one(data, len, pf);
    if (info) *info = pf.info;
    return rc;
}

int b200jpg_exif_orientation(const uint8_t *data, size_t len) {
    ParsedFrame pf;
    const int rc = parse_one(data, len, pf);
    return rc != 0 ? rc : pf.orientation;
}

int b200jpg_colorspace(const uint8_t *data, size_t len) {
    ParsedFrame pf;
    const int rc = parse_one(data, len, pf);
    return rc != 0 ? rc : frame_colorspace(pf);
}

int b200jpg_output_size(const uint8_t *data, size_t len, unsigned flags, uint32_t *width, uint32_t *height) {
    if (!width || !height) return B200JPG_ERR_INVALID_PARAMETER;
    ParsedFrame pf;
    const int rc = parse_one(data, len, pf);
    if (rc != 0) return rc;
    FramePlan p;
    p.k = downscale_of(flags);
    p.orientation = (flags & B200JPG_FLAG_EXIF_ORIENTATION) ? pf.orientation : 1;
    const Extent e = out_extent(pf.info, 0, flags & ~B200JPG_FLAG_NO_UPSAMPLE, p);
    *width = (uint32_t)e.w;
    *height = (uint32_t)e.h;
    return B200JPG_OK;
}

int b200jpg_draft_scale(const uint8_t *data, size_t len, uint32_t width, uint32_t height) {
    if (width == 0 || height == 0) return B200JPG_ERR_INVALID_PARAMETER;
    ParsedFrame pf;
    const int rc = parse_one(data, len, pf);
    return rc != 0 ? rc : (int)draft_scale_of(pf.info, width, height);
}

// the tables of resample_coefficients copied out (b200jpg_resample_coefficients / _box)
static int coefficients_out(uint32_t in_size, const float *box, uint32_t out_size, int resample, int32_t *bounds, int32_t *coeffs,
                            uint64_t capacity, uint32_t *ksize) {
    const bool cv = !box && resample_cv(resample & ~(B200JPG_CV_TABLE_VERTICAL | B200JPG_CV_TABLE_LINEAR));
    if (!ksize || in_size == 0 || out_size == 0 || !(resample_known(resample) || cv)) return B200JPG_ERR_INVALID_PARAMETER;
    std::vector<int32_t> b, k;
    uint32_t ks = 0;
    try {
        if (int rc = cv ? cv_resample_coefficients(in_size, out_size, resample, b, k, ks) : resample_coefficients(in_size, box, out_size, resample, b, k, ks))
            return rc;
    } catch (const std::bad_alloc &) {
        return B200JPG_ERR_OUT_OF_MEMORY;
    }
    *ksize = ks;
    if (!bounds || !coeffs) return B200JPG_OK;
    if (capacity < (uint64_t)out_size * ks) return B200JPG_ERR_INVALID_PARAMETER;
    memcpy(bounds, b.data(), b.size() * sizeof(int32_t));
    memcpy(coeffs, k.data(), k.size() * sizeof(int32_t));
    return B200JPG_OK;
}

int b200jpg_resample_coefficients(uint32_t in_size, uint32_t out_size, int resample, int32_t *bounds, int32_t *coeffs, uint64_t capacity,
                                  uint32_t *ksize) {
    return coefficients_out(in_size, nullptr, out_size, resample, bounds, coeffs, capacity, ksize);
}

int b200jpg_resample_coefficients_box(uint32_t in_size, float in0, float in1, uint32_t out_size, int resample, int32_t *bounds,
                                      int32_t *coeffs, uint64_t capacity, uint32_t *ksize) {
    if (!(in0 >= 0.0f && in0 <= in1 && in1 <= (float)in_size)) return B200JPG_ERR_INVALID_PARAMETER;  // (NaN fails too)
    const float box[2] = {in0, in1};
    return coefficients_out(in_size, box, out_size, resample, bounds, coeffs, capacity, ksize);
}

uint64_t b200jpg_build_tables(const uint8_t *data, size_t len, int scan, uint8_t *dst, uint64_t capacity) {
    ParsedFrame pf;
    std::string err;
    TableSet ts;
    int rc;
    try {
        rc = parse_codestream(data, len, pf, err);
        if (rc == 0 && (scan < 0 || scan >= (int)pf.scans.size())) {
            rc = B200JPG_ERR_INVALID_PARAMETER;
            err = "scan index out of range";
        }
        if (rc == 0) rc = build_table_set(pf.scans[scan], ts, err);
    } catch (const std::bad_alloc &) {
        rc = B200JPG_ERR_OUT_OF_MEMORY;
        err = "out of memory while building the decoder tables";
    }
    g_tls_code = rc;
    g_tls_error = err;
    if (rc) return 0;
    if (dst && capacity >= ts.blob.size()) memcpy(dst, ts.blob.data(), ts.blob.size());
    return ts.blob.size();
}

int b200jpg_create(int device, b200jpg_ctx **out) {
    if (!out) return B200JPG_ERR_INVALID_PARAMETER;
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        g_tls_code = B200JPG_ERR_NO_DEVICE;
        g_tls_error = "no CUDA device available: the H100 JPEG decode path has no CPU fallback";
        return B200JPG_ERR_NO_DEVICE;
    }
    if (device < 0) {
        e = cudaGetDevice(&device);
        if (e != cudaSuccess) device = 0;
    }
    if (device >= count) {
        g_tls_code = B200JPG_ERR_INVALID_PARAMETER;
        g_tls_error = "CUDA device ordinal out of range";
        return B200JPG_ERR_INVALID_PARAMETER;
    }
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess || prop.major != 9 || prop.minor != 0) {
        g_tls_code = B200JPG_ERR_NO_DEVICE;
        g_tls_error = "device is not a Hopper (sm_90a) GPU: the kernels are built for sm_90a only";
        return B200JPG_ERR_NO_DEVICE;
    }
    auto *c = new b200jpg_ctx();
    c->device = device;
    *out = c;
    return B200JPG_OK;
}

void b200jpg_destroy(b200jpg_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    ctx->trim();
    delete ctx;
}

void b200jpg_trim(b200jpg_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    ctx->trim();
}

int b200jpg_last_error(b200jpg_ctx *ctx, const char **message) {
    if (ctx) {
        if (message) *message = ctx->error.c_str();
        return ctx->code;
    }
    if (message) *message = g_tls_error.c_str();
    return g_tls_code;
}

void b200jpg_batch_destroy(b200jpg_batch *b) {
    if (!b) return;
    cudaSetDevice(b->ctx->device);
    if (b->ev_last) {  // buffers go back to the pool: nothing of this batch may still be in flight
        cudaEventSynchronize(b->ev_last);
        cudaEventDestroy(b->ev_last);
    }
    b->ctx->put(0, b->h_input, b->input_bytes);
    b->ctx->put(1, b->d_input, b->input_bytes);
    b->ctx->put(1, b->d_coef, b->coef_elems * sizeof(int16_t));
    b->ctx->put(1, b->d_samples, b->sample_elems * sizeof(int32_t));
    b->ctx->put(1, b->d_samples16, b->sample_elems * sizeof(int16_t));
    if (b->d_planes8) b->ctx->put(1, b->d_planes8, b->plane8_bytes);
    b->ctx->put(1, b->d_clean, b->clean_bytes);
    b->ctx->put(1, b->d_interval_len, b->sz_ilen);
    b->ctx->put(1, b->d_overrun, b->sz_overrun);
    if (b->d_spec) b->ctx->put(1, b->d_spec, b->sz_spec);
    if (b->d_dcplane) b->ctx->put(1, b->d_dcplane, b->coef_elems / 64 * sizeof(int16_t));
    b->ctx->put(1, b->d_status, b->sz_status);
    b->ctx->put(0, b->h_planes, b->slot_bytes() * b200jpg_batch::kPlaneSlots);
    b->ctx->put(1, b->d_planes, b->slot_bytes());
    if (b->d_scratch) b->ctx->put(1, b->d_scratch, b->scratch_bytes);
    if (b->d_inter) b->ctx->put(1, b->d_inter, b->inter_bytes);
    for (auto &e : b->ev_planes)
        if (e) cudaEventDestroy(e);
    for (auto &e : b->ev)
        if (e) cudaEventDestroy(e);
    delete b;
}

// ---- batch planning: the steps of batch_create_impl, in the order they run

// the caller's codestreams, then the residual codestreams of its JPEG XT frames, and why each frame failed
struct Codestreams {
    std::vector<const uint8_t *> data;
    std::vector<size_t> len;
    std::vector<std::string> err;
};

static void parse_frames(b200jpg_batch &b, Codestreams &cs, bool device_index) {
    b.frames.resize(b.n);
    b.parse_status.assign(b.n, 0);
    for_frames(b.n, 16, [&](int i) {
        try {  // an exception must not leave the thread (std::terminate): it fails this frame only
            b.parse_status[i] = parse_codestream(cs.data[i], cs.len[i], b.frames[i], cs.err[i], device_index);
        } catch (const std::bad_alloc &) {
            b.parse_status[i] = B200JPG_ERR_OUT_OF_MEMORY;
            cs.err[i] = "out of memory while parsing the codestream";
        } catch (...) {
            b.parse_status[i] = B200JPG_ERR_MALFORMED_STREAM;
            cs.err[i] = "codestream could not be parsed";
        }
    });
}

// JPEG XT (SURVEY 8f3): the residual codestream of a frame is one more frame of the batch -- same entropy kernels, same
// IDCT -- that owns no output; the parent's reconstruction merges the two (generic_reconstruct_kernel)
static void attach_residuals(b200jpg_batch &b, Codestreams &cs, bool device_index) {
    const int n_user = b.n_user;
    b.xt_child.assign(n_user, -1);
    for (int i = 0; i < n_user; i++) {
        if (b.parse_status[i] == 0 && !size_empty(b.plan[i].target) && b.frames[i].info.precision != 8) {
            b.parse_status[i] = B200JPG_ERR_NOT_IMPLEMENTED;  // never written unresized
            cs.err[i] = "only 8-bit frames are resized";
            continue;
        }
        if (b.parse_status[i] == 0 && (b.flags & kOutputModes) && frame_colorspace(b.frames[i]) == B200JPG_COLORSPACE_UNKNOWN) {
            b.parse_status[i] = B200JPG_ERR_NOT_IMPLEMENTED;  // never written with its own components
            cs.err[i] = "an output mode takes grey, YCbCr, RGB, and 8-bit Adobe CMYK or YCCK frames";
            continue;
        }
        // (a four-component frame that reaches this under a mode is 8-bit Adobe CMYK or YCCK: the check above refused the rest)
        const int nc = b.frames[i].info.ncomp;
        if (b.parse_status[i] == 0 && (b.flags & B200JPG_FLAG_LIBJPEG_TURBO) &&
            (b.frames[i].info.precision != 8 || (nc != 1 && nc != 3 && !(nc == 4 && (b.flags & kOutputModes))))) {
            b.parse_status[i] = B200JPG_ERR_NOT_IMPLEMENTED;
            cs.err[i] = "B200JPG_FLAG_LIBJPEG_TURBO takes 8-bit frames of one or three components, and Adobe CMYK or YCCK frames under an output mode";
            continue;
        }
        // libjpeg-turbo decodes the base codestream of a JPEG XT frame alone: no residual frame
        if (b.parse_status[i] != 0 || !b.frames[i].xt.present || (b.flags & B200JPG_FLAG_LIBJPEG_TURBO)) continue;
        if (b.flags & (B200JPG_FLAG_NO_COLOR_TRANSFORM | B200JPG_FLAG_NO_UPSAMPLE)) {
            b.parse_status[i] = B200JPG_ERR_NOT_IMPLEMENTED;
            cs.err[i] = "JPEG XT frames are only reconstructed with upsampling and colour transformation";
            continue;
        }
        if (downscale_of(b.flags) > 1) {  // never decoded base-only: the merge at reduced size is not defined here
            b.parse_status[i] = B200JPG_ERR_NOT_IMPLEMENTED;
            cs.err[i] = "JPEG XT frames are only reconstructed at full size";
            continue;
        }
        ParsedFrame rf;
        std::string rerr;
        const int rst = parse_residual(b.frames[i], rf, rerr, device_index);
        if (rst != 0) {
            b.parse_status[i] = rst;
            cs.err[i] = rerr;
            continue;
        }
        b.xt_child[i] = (int)b.frames.size();
        cs.data.push_back(b.frames[i].xt.resi.data());  // (the vectors' buffers stay where they are when b.frames grows: moved, not copied)
        cs.len.push_back(b.frames[i].xt.resi.size());
        b.frames.push_back(std::move(rf));
        b.parse_status.push_back(0);
        cs.err.emplace_back();
    }
    for (int i = 0; i < n_user; i++)  // push_back may have moved the frames: take the addresses again
        if (b.xt_child[i] >= 0) cs.data[b.xt_child[i]] = b.frames[i].xt.resi.data();
    b.n = (int)b.frames.size();
    b.plan.resize(b.n);
    b.xt_parent.assign(b.n, -1);
    for (int i = 0; i < n_user; i++)
        if (b.xt_child[i] >= 0) b.xt_parent[b.xt_child[i]] = i;
}

// What the kernels cover, and the decoder tables of every scan of the frames that pass. A frame that fails here fails the batch
// unless tolerate_bad: returns 0 or the status the batch fails with.
static int admit_frames(b200jpg_batch &b, Codestreams &cs, bool tolerate_bad, std::vector<std::vector<TableSet>> &frame_tables) {
    const int n = b.n;
    frame_tables.assign(n, {});
    TableCache table_cache;
    for (int i = 0; i < n; i++) {
        ParsedFrame &pf = b.frames[i];
        int &st = b.parse_status[i];
        if (st == 0) {
            const b200jpg_frame_info &fi = pf.info;
            bool factors_ok = fi.ncomp >= 1 && fi.ncomp <= 4;
            for (int c = 0; c < fi.ncomp; c++) factors_ok = factors_ok && fi.subx[c] >= 1 && fi.subx[c] <= 4 && fi.suby[c] >= 1 && fi.suby[c] <= 4;
            if (!factors_ok) {  // the reference's upsampler cores exist for factors 1..4 (upsampling/upsamplerbase.cpp:CreateUpsampler)
                st = B200JPG_ERR_NOT_IMPLEMENTED;
                cs.err[i] = "only frames of one to four components with subsampling factors of one to four are supported";
            } else {
                // A sequential frame codes a component at most once. A component no scan codes (the stream ends early: the
                // reference just stops at the EOI / the end of the data, Frame::ParseTrailer marker/frame.cpp:1062-1092)
                // keeps zero coefficients: the coefficient store is cleared for such batches. So do the blocks a single-component
                // scan leaves out: it codes the component's own block grid, ceil(ceil(W * h / hmax) / 8) x ceil(ceil(H * v / vmax)
                // / 8) (T.81 A.2.2), which can be smaller than the MCU-padded grid the store keeps (Y 3 x 3 next to 1 x 1 chroma,
                // 517 pixels wide: 65 of 66 block columns).
                int seen[4] = {0, 0, 0, 0};
                uint32_t hmax = 1, vmax = 1;
                for (int c = 0; c < fi.ncomp; c++) hmax = std::max<uint32_t>(hmax, fi.hs[c]), vmax = std::max<uint32_t>(vmax, fi.vs[c]);
                for (auto &sc : pf.scans) {
                    for (int k = 0; k < sc.ns; k++) seen[sc.comp[k]]++;
                    if (sc.ns == 1) {
                        const int c = sc.comp[0];
                        const uint32_t own_w = ((fi.width * fi.hs[c] + hmax - 1) / hmax + 7) / 8, own_h = ((fi.height * fi.vs[c] + vmax - 1) / vmax + 7) / 8;
                        if (own_w < fi.blocks_w[c] || own_h < fi.blocks_h[c]) b.clear_coef = true;
                    }
                }
                for (int c = 0; c < fi.ncomp; c++) {
                    if (fi.frame_type != 2 && seen[c] > 1) {
                        st = B200JPG_ERR_NOT_IMPLEMENTED;
                        cs.err[i] = "sequential frame codes a component more than once, not supported by the GPU path";
                    }
                    if (seen[c] == 0) b.clear_coef = true;
                }
            }
        }
        // all table sets of the frame before any of its scans joins a launch class: a frame that fails here must not leave
        // scans behind that decode bytes nobody uploads
        if (st == 0) {
            frame_tables[i].resize(pf.scans.size());
            for (size_t si = 0; si < pf.scans.size() && st == 0; si++) {
                try {
                    st = build_table_set_cached(pf.scans[si], frame_tables[i][si], cs.err[i], table_cache);
                } catch (const std::bad_alloc &) {
                    st = B200JPG_ERR_OUT_OF_MEMORY;
                    cs.err[i] = "out of memory while building the decoder tables";
                }
            }
        }
        if (st != 0 && b.xt_parent[i] >= 0) {  // a residual codestream the kernels do not cover fails its frame
            const int par = b.xt_parent[i];
            if (b.parse_status[par] == 0) b.parse_status[par] = st, cs.err[par] = "residual codestream: " + cs.err[i];
            b.xt_child[par] = -1;
            if (!tolerate_bad) return b.ctx->fail(st, "frame " + std::to_string(par) + ": " + cs.err[par]);
        }
        if (st != 0 && !tolerate_bad) return b.ctx->fail(st, "frame " + std::to_string(i) + ": " + cs.err[i]);
    }
    for (int i = 0; i < n; i++)  // ... and a frame that failed takes its residual codestream with it
        if (b.xt_parent[i] >= 0 && b.parse_status[b.xt_parent[i]] != 0 && b.parse_status[i] == 0) b.parse_status[i] = b.parse_status[b.xt_parent[i]];
    return B200JPG_OK;
}

// layout of the packed input buffer: [codestreams][table blobs][per class: scans, intervals][per group: frames]. Here the first
// region: returns the offset of every frame's codestream.
static std::vector<uint64_t> lay_out_codestreams(b200jpg_batch &b, const std::vector<size_t> &len) {
    std::vector<uint64_t> byte_off(b.n, 0);
    uint64_t cur = 0;
    for (int i = 0; i < b.n; i++) {
        byte_off[i] = cur;
        if (b.parse_status[i] == 0) cur = align_up(cur + len[i] + 32, 16);
    }
    b.bytes_region = align_up(cur + 64, 256);
    return byte_off;
}

// How live frame i is reconstructed. The tuned kernels cover 8-bit grey frames and three-component frames whose first component
// is not subsampled and whose two other components share factors of 1 or 2; everything else (SURVEY 8f4), planes without
// upsampling and both codestreams of a JPEG XT frame go through the generic kernels. Downscaled frames: 8-bit 4:2:0 frames with
// upsampling take reconstruct420_scaled_kernel, every other one the scaled IDCT into int32 planes and then the generic kernels (a
// JPEG XT frame never gets here downscaled: attach_residuals refuses it).
// B200JPG_FLAG_LIBJPEG_TURBO (8-bit grey and three-component frames, and CMYK / YCCK frames under a mode: attach_residuals): the
// tiled turbo_reconstruct_kernel covers component 0 at full resolution, alone or with two chroma components of equal factors 1 or
// 2 whose fancy upsampling has both neighbours (more than 2 chroma samples per row when halved horizontally); everything else,
// four-component frames always (DESIGN §18), the generic turbo kernel. ncomp: the
// components reconstructed (1 for mode "L" of a YCbCr frame). A frame drafted to 1/k (k > 1, DESIGN §17) is judged on the ratios
// after its IDCTs (draft_ratio) and its reduced width: its luma block is then 8 / k wide, and its chroma ratios 1 x 1 (4:4:4,
// 4:2:0), 2 x 1 (4:2:2) or 1 x 2 (4:4:0); 2 x 2 never occurs at k > 1 and is left to the generic kernel
static ReconPath turbo_path(const b200jpg_frame_info &fi, int ncomp, uint32_t k) {
    if (ncomp == 4 || fi.subx[0] != 1 || fi.suby[0] != 1) return ReconPath::TurboGeneric;  // (the tiled kernel has no fourth component)
    if (ncomp == 1) return ReconPath::Turbo;
    const Ratio r = draft_ratio(fi, 1, k), r2 = draft_ratio(fi, 2, k);
    if (r.x != r2.x || r.y != r2.y || r.x > 2 || r.y > 2) return ReconPath::TurboGeneric;
    if (k > 1 && (fi.hs[1] != fi.hs[2] || fi.vs[1] != fi.vs[2] || (r.x == 2 && r.y == 2))) return ReconPath::TurboGeneric;
    const uint32_t w = (fi.width + k - 1) / k;
    return (r.x == 2 && (w + 1) / 2 <= 2) ? ReconPath::TurboGeneric : ReconPath::Turbo;
}

static ReconPath recon_path(const b200jpg_batch &b, int i) {
    const b200jpg_frame_info &fi = b.frames[i].info;
    const bool scaled = b.plan[i].k > 1;
    if (b.flags & B200JPG_FLAG_LIBJPEG_TURBO) return turbo_path(fi, fi.ncomp, b.plan[i].k);
    if (b.xt_parent[i] >= 0 || (i < b.n_user && b.xt_child[i] >= 0)) return ReconPath::Generic;
    if (b.flags & B200JPG_FLAG_NO_UPSAMPLE) return scaled ? ReconPath::Scaled : ReconPath::Generic;  // planes of every component, then one sample -> one output value
    if (fi.precision != 8) return scaled ? ReconPath::Scaled : ReconPath::Generic;  // 12-bit frames: int32 planes, 16-bit samples out
    if (fi.ncomp == 1) return scaled ? ReconPath::Scaled : ((fi.subx[0] != 1 || fi.suby[0] != 1) ? ReconPath::Generic : ReconPath::Tiled);
    if (fi.ncomp != 3 || fi.subx[0] != 1 || fi.suby[0] != 1 || fi.subx[1] != fi.subx[2] || fi.suby[1] != fi.suby[2] || fi.subx[1] > 2 || fi.suby[1] > 2)
        return scaled ? ReconPath::Scaled : ReconPath::Generic;
    if (fi.subx[1] == 2 && fi.suby[1] == 2) return scaled ? ReconPath::Scaled420 : ReconPath::Fused420;
    return scaled ? ReconPath::Scaled : ReconPath::Tiled;
}

// The plan of the caller's live frame i as far as its factor k decides it (right after admit_drafts): the path, the components,
// the output mode and the orientation; the admission steps add the request
static void frame_plan(b200jpg_batch &b, int i) {
    const b200jpg_frame_info &fi = b.frames[i].info;
    FramePlan &p = b.plan[i];
    p.path = recon_path(b, i);
    p.ncomp = p.out_ncomp = fi.ncomp;
    p.orientation = (b.flags & B200JPG_FLAG_EXIF_ORIENTATION) ? b.frames[i].orientation : 1;
    if (size_empty(p.target)) p.orientation = kFlipOrientation[p.orientation - 1][p.flip];  // (DESIGN §21)
    const bool xt = b.xt_child[i] >= 0;
    if ((b.flags & B200JPG_FLAG_OUTPUT_L) && fi.ncomp == 3) {
        p.out_ncomp = 1;
        if (fi.ycbcr && !xt) {
            // luma alone: a grey frame over component 0 on the MCU-padded block grid; libjpeg's JCS_GRAYSCALE for YCbCr input
            p.ncomp = 1;
            if (b.flags & B200JPG_FLAG_LIBJPEG_TURBO) p.path = turbo_path(fi, 1, p.k);  // the turbo kernels over component 0
            else if (p.k > 1) p.path = ReconPath::Scaled;
            else p.path = (fi.precision != 8 || fi.subx[0] != 1 || fi.suby[0] != 1) ? ReconPath::Generic : ReconPath::Tiled;
        } else {  // RGB-coded and JPEG XT frames: the L formula after the colour transformation (merge) and clamp, in the generic kernels
            p.mode = OutMode::Luma;
            if (!(b.flags & B200JPG_FLAG_LIBJPEG_TURBO)) p.path = p.k > 1 ? ReconPath::Scaled : ReconPath::Generic;
        }
    }
    if ((b.flags & B200JPG_FLAG_OUTPUT_RGB) && fi.ncomp == 1) {
        p.out_ncomp = 3;
        p.mode = OutMode::Replicate;
    }
    if ((b.flags & kOutputModes) && fi.ncomp == 4) {  // CMYK / YCCK (attach_residuals refused the rest): all four reconstructed,
        const bool rgb = (b.flags & B200JPG_FLAG_OUTPUT_RGB) != 0;  // Pillow's conversion in the generic kernels (DESIGN §15, §18)
        p.out_ncomp = rgb ? 3 : 1;
        p.mode = rgb ? OutMode::CmykRgb : OutMode::CmykLuma;
        if (b.flags & B200JPG_FLAG_LIBJPEG_TURBO) p.path = ReconPath::TurboGeneric;
        else p.path = p.k > 1 ? ReconPath::Scaled : ReconPath::Generic;
    }
    p.described = p.orientation != 1 || p.mode != OutMode::Coded;  // (admit_crops adds the cropped frames)
}

// Coefficient, sample and output layout of the live frames; returns the sample plane offsets. The sample planes a frame gets
// follow its reconstruction path: Generic one per component, Tiled one per component from 1 on, Fused420 none (its chroma samples
// live in shared memory), Scaled one per component of 8 ceil(blocks_w / k) x 8 ceil(blocks_h / k) samples, Scaled420 none,
// TurboGeneric one uint8 plane per reconstructed component (s_c x s_c bytes per block of a drafted frame, draft_idct_size) and Turbo
// one per component from 1 on, byte offsets into the batch's uint8 plane buffer.
static std::vector<std::array<uint64_t, 4>> lay_out_planes(b200jpg_batch &b) {
    const int n = b.n;
    b.coef_base.assign(n, {});
    b.out_off.assign(n, 0);
    b.out_bytes.assign(n, 0);
    std::vector<std::array<uint64_t, 4>> sample_base(n);
    uint64_t coef_cur = 0, sample_cur = 0, out_cur = 0, plane8_cur = 0;
    for (int i = 0; i < n; i++) {
        if (b.parse_status[i] != 0) continue;
        const b200jpg_frame_info &fi = b.frames[i].info;
        const FramePlan &plan = b.plan[i];
        const ReconPath path = plan.path;
        const int first_plane = (path == ReconPath::Generic || path == ReconPath::Scaled || path == ReconPath::TurboGeneric) ? 0 : (path == ReconPath::Tiled ? 1 : fi.ncomp);
        const uint32_t k = plan.k;
        uint64_t samples = 0;
        for (int c = 0; c < fi.ncomp; c++) {  // every component is entropy decoded; only the reconstructed ones get sample planes
            const uint64_t elems = (uint64_t)fi.blocks_w[c] * fi.blocks_h[c] * 64;
            b.coef_base[i][c] = coef_cur;
            coef_cur += elems;
            if ((path == ReconPath::TurboGeneric || (path == ReconPath::Turbo && c >= 1)) && c < (int)plan.ncomp) {
                const uint64_t s = draft_idct_size(fi, c, k);  // s x s bytes per block (8 x 8 undrafted)
                sample_base[i][c] = plane8_cur;
                plane8_cur = align_up(plane8_cur + elems / 64 * s * s, 256);
            } else if (c >= first_plane && c < (int)plan.ncomp) {
                sample_base[i][c] = sample_cur;
                sample_cur += path == ReconPath::Scaled ? 64ull * ((fi.blocks_w[c] + k - 1) / k) * ((fi.blocks_h[c] + k - 1) / k) : elems;
            }
        }
        for (uint32_t c = 0; c < plan.out_ncomp; c++) {
            const Extent e = out_extent(fi, (int)c, b.flags, plan);  // the components one after the other
            samples += e.w * e.h;
        }
        b.out_off[i] = out_cur;
        b.out_bytes[i] = (b.xt_parent[i] >= 0) ? 0 : samples * (fi.precision > 8 ? 2u : 1u);  // a residual codestream has no pixels of its own
        out_cur = align_up(out_cur + b.out_bytes[i], 256);
        b.ecs_bytes += fi.ecs_bytes;
        b.stored_blocks += fi.stored_blocks;
    }
    b.out_total = out_cur;
    b.coef_elems = coef_cur;
    b.sample_elems = sample_cur;
    b.plane8_bytes = plane8_cur;
    return sample_base;
}

// table sets (deduplicated by content) and scan classes, launched in the order they are formed here except that the scans of a
// progressive frame build on each other: launch order = scan order (sequential classes: ordinal 0)
static void form_scan_classes(b200jpg_batch &b, std::vector<std::vector<TableSet>> &frame_tables, const std::vector<uint64_t> &byte_off) {
    std::map<std::vector<uint8_t>, int> table_index;
    std::map<ClassKey, int> class_index;
    for (int i = 0; i < b.n; i++) {
        if (b.parse_status[i] != 0) continue;
        ParsedFrame &pf = b.frames[i];
        const b200jpg_frame_info &fi = pf.info;
        for (size_t si = 0; si < pf.scans.size(); si++) {
            auto &sc = pf.scans[si];
            TableSet &ts = frame_tables[i][si];
            int ti;
            auto it = table_index.find(ts.blob);
            if (it == table_index.end()) {
                ti = (int)b.table_sets.size();
                table_index.emplace(ts.blob, ti);
                b.table_sets.push_back(std::move(ts));
            } else {
                ti = it->second;
            }
            ScanClassParams p{};
            p.ns = sc.ns;
            for (int k = 0; k < sc.ns; k++) {
                int ci = sc.comp[k];
                p.mw[k] = (sc.ns > 1) ? fi.hs[ci] : 1;
                p.mh[k] = (sc.ns > 1) ? fi.vs[ci] : 1;
                p.bw[k] = (int)fi.blocks_w[ci];
                p.dc_slot[k] = sc.td[k];
                p.ac_slot[k] = sc.ta[k];
                p.q_slot[k] = fi.tq[ci];
            }
            p.mcu_cols = sc.mcu_cols;
            p.total_mcus = sc.mcu_cols * sc.mcu_rows;
            p.dri = sc.dri ? sc.dri : p.total_mcus;
            p.intervals_per_scan = (uint32_t)sc.interval_off.size();
            p.lut_words = b.table_sets[ti].lut_words();
            p.progressive = sc.progressive ? 1 : 0;
            p.ss = sc.ss;
            p.se = sc.se;
            p.ah = sc.ah;
            p.al = sc.lowbit;
            p.ordinal = sc.progressive ? (int)si : 0;
            p.indexed = sc.spec ? 1 : 0;
            const ClassKey key{p, ti};  // n_scans and segs_per_scan are still 0 here
            int cidx;
            auto cit = class_index.find(key);
            if (cit == class_index.end()) {
                cidx = (int)b.classes.size();
                class_index.emplace(key, cidx);
                ScanClass cl;
                cl.p = p;
                cl.table_set = ti;
                b.classes.push_back(std::move(cl));
            } else {
                cidx = cit->second;
            }
            ScanClass &cl = b.classes[cidx];
            cl.frame_comp0 = sc.comp[0];
            ClassScan cs{};
            for (int k = 0; k < sc.ns; k++) cs.coef_base[k] = b.coef_base[i][sc.comp[k]];
            cs.frame = (uint32_t)i;
            cl.scans.push_back(cs);
            cl.scan_on_device.push_back(sc.device_index ? 1 : 0);
            cl.scan_ecs_off.push_back(byte_off[i] + (uint64_t)sc.ecs_off);
            cl.scan_ecs_end.push_back(byte_off[i] + (uint64_t)sc.ecs_end);
            if (sc.spec) {  // work items per scan: what the longest scan of the class needs (unstuffing only shrinks the data)
                const uint32_t need = (uint32_t)(((uint64_t)(sc.ecs_end - sc.ecs_off) * 8u + kSpecSeqBits - 1u) / kSpecSeqBits) + 1u;
                cl.p.segs_per_scan = std::max(cl.p.segs_per_scan, need);
            }
            for (size_t k = 0; k < sc.interval_off.size(); k++) {
                size_t off = sc.interval_off[k], end = sc.interval_end[k];
                cl.interval_off.push_back(off == SIZE_MAX ? ~0ull : byte_off[i] + (uint64_t)off);
                uint64_t e = off == SIZE_MAX ? 0ull : byte_off[i] + (uint64_t)end;
                // the data ends inside the scan's last interval: flagged for the decoder (kIntervalEofFlag)
                if (sc.eof_tail && off != SIZE_MAX && k + 1 == sc.interval_off.size()) e |= kIntervalEofFlag;
                cl.interval_end.push_back(e);
            }
        }
    }
    std::stable_sort(b.classes.begin(), b.classes.end(), [](const ScanClass &x, const ScanClass &y) { return x.p.ordinal < y.p.ordinal; });
}

// Component-fused progressive groups: classes that hold exactly the same frames in the same order and whose scans are either
// interleaved DC scans of all components or single-component AC scans with equal restart intervals per group. The other
// progressive frames go scan by scan and are dequantised after their last scan.
static void form_progressive_groups(b200jpg_batch &b) {
    std::vector<uint8_t> frame_fused(b.n, 0);
    if (getenv("B200JPG_NO_PFUSE") == nullptr) {
        std::map<std::vector<uint32_t>, std::vector<int>> by_frames;
        for (size_t ci = 0; ci < b.classes.size(); ci++) {
            const ScanClass &cl = b.classes[ci];
            if (!cl.p.progressive) continue;
            std::vector<uint32_t> ids;
            for (auto &cs : cl.scans) ids.push_back(cs.frame);
            by_frames[ids].push_back((int)ci);
        }
        for (auto &kv : by_frames) {
            const std::vector<uint32_t> &ids = kv.first;
            std::vector<int> cls = kv.second;  // ascending ordinal (the classes are sorted)
            bool ok = !ids.empty();
            for (uint32_t id : ids) ok = ok && b.frames[id].scans.size() == cls.size();
            PfGroupHost grp;
            const ParsedFrame &pf0 = b.frames[ids[0]];
            const b200jpg_frame_info &fi0 = pf0.info;
            // one DC quantiser per component serves the whole group
            for (uint32_t id : ids)
                for (int c = 0; c < fi0.ncomp; c++) ok = ok && b.frames[id].comp_quant[c][0] == pf0.comp_quant[c][0];
            for (int ci : cls) {
                const ScanClassParams &p = b.classes[(size_t)ci].p;
                if (!ok) break;
                if (p.ss == 0) {
                    ok = p.ns == (int)fi0.ncomp && (grp.dc.empty() ? p.ah == 0 : p.ah != 0);
                    if (ok && !grp.dc.empty()) {
                        const ScanClassParams &q = b.classes[(size_t)grp.dc[0]].p;
                        ok = q.dri == p.dri && q.intervals_per_scan == p.intervals_per_scan && q.total_mcus == p.total_mcus;
                    }
                    grp.dc.push_back(ci);
                } else {
                    const int c = b.classes[(size_t)ci].frame_comp0;
                    ok = p.ns == 1 && c < 4;
                    if (ok && !grp.ac[c].empty()) {
                        const ScanClassParams &q = b.classes[(size_t)grp.ac[c][0]].p;
                        ok = q.dri == p.dri && q.intervals_per_scan == p.intervals_per_scan && q.total_mcus == p.total_mcus && q.mcu_cols == p.mcu_cols;
                    }
                    if (ok) grp.ac[c].push_back(ci);
                }
            }
            ok = ok && !grp.dc.empty() && grp.dc.size() <= (size_t)kPfMaxScans;
            for (int c = 0; c < 4; c++) ok = ok && grp.ac[c].size() <= (size_t)kPfMaxScans;
            if (!ok) continue;
            for (int ci : cls) b.classes[(size_t)ci].fused = true;
            for (uint32_t id : ids) frame_fused[id] = 1;
            for (int c = 0; c < 4; c++) b.pf_dc_quant.push_back(c < fi0.ncomp ? pf0.comp_quant[c][0] : 0);
            b.pf_groups.push_back(std::move(grp));
        }
    }
    for (int i = 0; i < b.n; i++) {
        if (b.parse_status[i] != 0 || b.frames[i].info.frame_type != 2 || frame_fused[i]) continue;
        const ParsedFrame &pf = b.frames[i];
        ProgFrame f{};
        f.frame = (uint32_t)i;
        for (int c = 0; c < pf.info.ncomp; c++) {
            f.coef_base[c] = b.coef_base[i][c];
            f.n_blocks[c] = pf.info.blocks_w[c] * pf.info.blocks_h[c];
            b.prog_max_blocks = std::max(b.prog_max_blocks, f.n_blocks[c]);
            for (int k = 0; k < 64; k++) f.q_raster[c][kZigZagToRaster[k]] = pf.comp_quant[c][k];
        }
        b.prog_frames.push_back(f);
    }
}

// Unstuffed-buffer layout. Host-indexed scans: every interval gets its source length rounded up to 16 bytes + 48 bytes of zero
// tail. Device-indexed scans: one region of ECS length + kCleanSlackPerInterval per interval, inside which the index kernel places
// interval k at (its source offset) + kCleanSlackPerInterval * k -- no lengths are known here.
static void lay_out_unstuffed(b200jpg_batch &b) {
    uint64_t ccur = 0, ibase = 0;
    for (size_t ci = 0; ci < b.classes.size(); ci++) {
        auto &cl = b.classes[ci];
        cl.p.n_scans = (uint32_t)cl.scans.size();
        cl.interval_base = ibase;
        cl.clean_off.resize(cl.interval_off.size());
        const size_t nint = cl.p.intervals_per_scan;
        for (size_t j = 0; j < cl.scans.size(); j++) {
            if (cl.scan_on_device[j]) {
                IndexScan is{};
                is.ecs_off = cl.scan_ecs_off[j];
                is.ecs_end = cl.scan_ecs_end[j];
                is.off_arr = (uint64_t)ci;  // class index for now: becomes the array offset once the layout is known
                is.end_arr = (uint64_t)(j * nint);
                is.clean_base = ccur;
                is.n_intervals = (uint32_t)nint;
                is.frame = cl.scans[j].frame;
                b.index_scans.push_back(is);
                for (size_t k = 0; k < nint; k++) cl.clean_off[j * nint + k] = ccur;
                ccur += align_up((is.ecs_end - is.ecs_off) + (uint64_t)kCleanSlackPerInterval * nint + 64, 16);
            } else {
                for (size_t k = j * nint; k < (j + 1) * nint; k++) {
                    cl.clean_off[k] = ccur;
                    uint64_t len = cl.interval_off[k] == ~0ull ? 0 : (cl.interval_end[k] & ~kIntervalEofFlag) - cl.interval_off[k];
                    ccur += align_up(len, 16) + 48;
                }
            }
        }
        ibase += cl.interval_off.size();
        if (cl.p.indexed) {
            cl.spec_base = b.n_spec;
            b.n_spec += (uint64_t)cl.scans.size() * cl.p.segs_per_scan;
        }
    }
    b.clean_bytes = ccur + 512;  // slack: the ring prefetch runs up to 64 bytes ahead of the reader
    b.n_intervals = ibase;
}

// Reconstruction groups: frames of one component count, chroma factors and reconstruction path share the launches
static void form_recon_groups(b200jpg_batch &b, const std::vector<std::array<uint64_t, 4>> &sample_base) {
    for (int i = 0; i < b.n; i++) {
        if (b.parse_status[i] != 0) continue;
        const b200jpg_frame_info &fi = b.frames[i].info;
        const int xt_res = (i < b.n_user) ? b.xt_child[i] : -1;  // JPEG XT: this frame's residual frame
        const FramePlan &plan = b.plan[i];
        const ReconPath path = plan.path;
        const uint32_t nc = plan.ncomp, k = plan.k;
        const bool generic = path == ReconPath::Generic || path == ReconPath::Scaled || path == ReconPath::TurboGeneric;
        uint32_t sx = nc > 1 ? fi.subx[1] : 1, sy = nc > 1 ? fi.suby[1] : 1;
        if (nc > 1 && path == ReconPath::Turbo) sx = draft_ratio(fi, 1, k).x, sy = draft_ratio(fi, 1, k).y;
        if (generic) sx = sy = 0;  // one group per component count: the generic kernels read the factors per frame
        // oriented frames (B200JPG_FLAG_EXIF_ORIENTATION, 2..8) form groups of their own, one per orientation: their destinations
        // are rewritten descriptors, whose store kind is chosen per group. Cropped frames too: their launches are sized by the tiles
        // the rectangles cover, and they always store clipped. Resized frames too (every one of them is cropped, admit_crops): they
        // store into the scratch, unconverted. And the frames of an output mode, keyed by it, and of one scale: a group's launches
        // take its factor k. A resized grey frame of B200JPG_FLAG_OUTPUT_RGB writes its one channel into the scratch: the resample
        // pass replicates it
        const OutMode mode = (plan.resized && plan.mode == OutMode::Replicate) ? OutMode::Coded : plan.mode;
        const GroupKey key{nc, sx, sy, path, plan.orientation, plan.cropped, plan.resized, plan.described, mode, k};
        b.rewritten = b.rewritten || plan.described;
        ReconGroup *g = nullptr;
        for (auto &gg : b.groups)
            if (gg.key == key) g = &gg;
        if (!g) {
            b.groups.emplace_back();
            g = &b.groups.back();
            g->key = key;
        }
        FrameRecon fr{};
        const bool drafted = k > 1 && (path == ReconPath::TurboGeneric || path == ReconPath::Turbo);
        uint32_t hmax = 1, vmax = 1;
        for (int c = 0; c < fi.ncomp; c++) hmax = std::max<uint32_t>(hmax, fi.hs[c]), vmax = std::max<uint32_t>(vmax, fi.vs[c]);
        for (uint32_t c = 0; c < nc; c++) {
            fr.coef_base[c] = b.coef_base[i][c];
            fr.sample_base[c] = sample_base[i][c];
            fr.bw[c] = fi.blocks_w[c];
            fr.bh[c] = fi.blocks_h[c];
            fr.csx[c] = fi.subx[c];
            fr.csy[c] = fi.suby[c];
            if (drafted) {  // the coefficient grid on both sides, s x s samples per block, the ratios after the reduced IDCT
                const uint32_t s = draft_idct_size(fi, (int)c, k);
                fr.coef_bw[c] = fi.blocks_w[c];
                fr.coef_bh[c] = fi.blocks_h[c];
                fr.idct[c] = (uint8_t)s;
                fr.csx[c] = (uint8_t)(hmax * (8 / k) / (fi.hs[c] * s));
                fr.csy[c] = (uint8_t)(vmax * (8 / k) / (fi.vs[c] * s));
            } else if (k > 1) {  // the grid of the reduced planes; the coefficient grid moves to coef_bw / coef_bh
                fr.coef_bw[c] = fi.blocks_w[c];
                fr.coef_bh[c] = fi.blocks_h[c];
                fr.bw[c] = (fi.blocks_w[c] + k - 1) / k;
                fr.bh[c] = (fi.blocks_h[c] + k - 1) / k;
            }
        }
        fr.fancy = k < 8;  // libjpeg-turbo upsamples by replication at 1/8 (min_DCT_scaled_size == 1)
        fr.out_base = b.out_off[i];
        const Extent reduced = decoded_extent(fi, 0, b.flags & ~B200JPG_FLAG_NO_UPSAMPLE, k);  // W' x H' (the full size at k = 1)
        fr.width = (uint32_t)reduced.w;
        fr.height = (uint32_t)reduced.h;
        if (b.xt_parent[i] >= 0) fr.width = fr.height = 0;  // a residual codestream: planes only, its frame's reconstruction reads them
        if (xt_res >= 0) {
            const b200jpg_frame_info &ri = b.frames[xt_res].info;
            fr.xt = 1u | (b.frames[i].xt.l_ycbcr ? 2u : 0u) | (b.frames[i].xt.r_ycbcr ? 4u : 0u);
            for (int c = 0; c < ri.ncomp; c++) {
                fr.res_sample_base[c] = sample_base[xt_res][c];
                fr.res_bw[c] = ri.blocks_w[c];
                fr.res_csx[c] = ri.subx[c];
                fr.res_csy[c] = ri.suby[c];
            }
        }
        fr.ncomp = nc;
        fr.ycbcr = (b.flags & B200JPG_FLAG_NO_COLOR_TRANSFORM) ? 0 : fi.ycbcr;  // JPGTAG_MATRIX_LTRAFO = ..._NONE (rectanglerequest.cpp:150-152)
        // CMYK and YCCK frames of an output mode share their groups: the YCC -> RGB step is a per-frame switch
        fr.ycck = (plan.mode == OutMode::CmykRgb || plan.mode == OutMode::CmykLuma) && frame_colorspace(b.frames[i]) == B200JPG_COLORSPACE_YCCK;
        fr.subx = sx;
        fr.suby = sy;
        fr.cw = (uint32_t)(sx ? (reduced.w + sx - 1) / sx : reduced.w);  // (generic groups carry the factors per component: csx / csy)
        fr.ch = (uint32_t)(sy ? (reduced.h + sy - 1) / sy : reduced.h);
        fr.status_idx = (uint32_t)i;
        fr.precision = fi.precision;
        if (plan.cropped) {
            // the tiles of the path that cover the clip rectangle, from tile (tx0, ty0) on; the launch grid is sized by the largest
            // such range of the group and every CTA runs tile (tx0 + bx, ty0 + by) exactly as the uncropped decode does
            const Clip cl = crop_to_decoded(plan.orientation, plan.crop, reduced.w, reduced.h);
            const ReconTile t = recon_tile(path);
            const uint32_t bpx = (drafted && path == ReconPath::Turbo) ? 8 / k : 8;  // output pixels per tile block: a drafted luma block's
            const uint32_t tw = bpx * t.bw, th = bpx * t.bh;
            fr.clip_x0 = cl.x0, fr.clip_y0 = cl.y0, fr.clip_x1 = cl.x1, fr.clip_y1 = cl.y1;
            fr.tx0 = cl.x0 / tw, fr.ty0 = cl.y0 / th;
            const uint32_t ntx = (cl.x1 - 1) / tw - fr.tx0 + 1, nty = (cl.y1 - 1) / th - fr.ty0 + 1;
            if (drafted && path == ReconPath::Turbo && nc > 1) {
                // the chroma samples under those tiles, one more on each side (the upsampling window), as blocks of idct[1] samples
                const int64_t s = fr.idct[1];
                const int64_t jx0 = (int64_t)fr.tx0 * tw / sx - 1, jy0 = (int64_t)fr.ty0 * th / sy - 1;
                const int64_t jx1 = ((int64_t)(fr.tx0 + ntx) * tw - 1) / sx + 1, jy1 = ((int64_t)(fr.ty0 + nty) * th - 1) / sy + 1;
                fr.cb_x0 = (uint32_t)(std::max<int64_t>(jx0, 0) / s), fr.cb_y0 = (uint32_t)(std::max<int64_t>(jy0, 0) / s);
                fr.cb_x1 = (uint32_t)std::min<int64_t>(jx1 / s + 1, fi.blocks_w[1]), fr.cb_y1 = (uint32_t)std::min<int64_t>(jy1 / s + 1, fi.blocks_h[1]);
                g->max_bwc = std::max(g->max_bwc, fr.cb_x1 - fr.cb_x0);
                g->max_bhc = std::max(g->max_bhc, fr.cb_y1 - fr.cb_y0);
            } else if ((path == ReconPath::Tiled || path == ReconPath::Turbo) && nc > 1) {
                // b1: the chroma blocks under those tiles, one more on each side (the upsampling window), clipped to the plane
                const int64_t cbx0 = (int64_t)fr.tx0 * t.bw / sx - 1, cby0 = (int64_t)fr.ty0 * t.bh / sy - 1;
                const int64_t cbx1 = (int64_t)(fr.tx0 + ntx) * t.bw / sx + 1, cby1 = (int64_t)(fr.ty0 + nty) * t.bh / sy + 1;
                fr.cb_x0 = (uint32_t)std::max<int64_t>(cbx0, 0), fr.cb_y0 = (uint32_t)std::max<int64_t>(cby0, 0);
                fr.cb_x1 = (uint32_t)std::min<int64_t>(cbx1, fi.blocks_w[1]), fr.cb_y1 = (uint32_t)std::min<int64_t>(cby1, fi.blocks_h[1]);
                g->max_bwc = std::max(g->max_bwc, fr.cb_x1 - fr.cb_x0);
                g->max_bhc = std::max(g->max_bhc, fr.cb_y1 - fr.cb_y0);
            }
            g->max_bw0 = std::max(g->max_bw0, ntx * t.bw);
            g->max_bh0 = std::max(g->max_bh0, nty * t.bh);
        } else {
            g->max_bw0 = std::max(g->max_bw0, (uint32_t)(reduced.w + 7) / 8);
            g->max_bh0 = std::max(g->max_bh0, (uint32_t)(reduced.h + 7) / 8);
        }
        g->frames.push_back(fr);
        if (generic) {  // the largest block grid of any component: the extent of the generic (or scaled) IDCT launch
            for (uint32_t c = 0; c < nc; c++)
                if ((uint64_t)fi.blocks_w[c] * fi.blocks_h[c] > (uint64_t)g->max_bwc * g->max_bhc) g->max_bwc = fi.blocks_w[c], g->max_bhc = fi.blocks_h[c];
        } else if (nc > 1 && !plan.cropped) {  // (a cropped Tiled frame: its chroma block range above)
            g->max_bwc = std::max(g->max_bwc, fi.blocks_w[1]);
            g->max_bhc = std::max(g->max_bhc, fi.blocks_h[1]);
        }
    }
}

// descriptor region of the input buffer, behind the codestreams
static void lay_out_descriptors(b200jpg_batch &b) {
    uint64_t cur = b.bytes_region;
    b.dev_tables.resize(b.table_sets.size());
    for (size_t t = 0; t < b.table_sets.size(); t++) {
        b.dev_tables[t] = cur;
        cur = align_up(cur + b.table_sets[t].blob.size(), 256);
    }
    for (auto &cl : b.classes) {
        cl.dev_scans = cur;
        cur = align_up(cur + cl.scans.size() * sizeof(ClassScan), 256);
        cl.dev_intervals = cur;
        cur = align_up(cur + cl.interval_off.size() * sizeof(uint64_t), 256);
        cl.dev_interval_end = cur;
        cur = align_up(cur + cl.interval_end.size() * sizeof(uint64_t), 256);
        cl.dev_clean_off = cur;
        cur = align_up(cur + cl.clean_off.size() * sizeof(uint64_t), 256);
    }
    for (auto &g : b.groups) {
        g.dev_frames = cur;
        cur = align_up(cur + g.frames.size() * sizeof(FrameRecon), 256);
    }
    b.dev_rs_frames = cur;
    cur = align_up(cur + b.rs_frames.size() * sizeof(ResampleFrame), 256);
    for (size_t r = 0; r < b.rs_frames.size(); r++) {  // the tables, 16-byte aligned and padded (resample_h_kernel stages them in uint4)
        ResampleFrame &f = b.rs_frames[r];
        uint64_t *at[4] = {&f.h_bounds, &f.h_coef, &f.v_bounds, &f.v_coef};
        for (int t = 0; t < 4; t++) {
            *at[t] = cur;
            cur = align_up(cur + b.rs_tables[r][t].size() * sizeof(int32_t), 16);
        }
    }
    cur = align_up(cur, 256);
    b.dev_prog_frames = cur;
    cur = align_up(cur + b.prog_frames.size() * sizeof(ProgFrame), 256);
    b.dev_index_scans = cur;
    cur = align_up(cur + b.index_scans.size() * sizeof(IndexScan), 256);
    for (auto &is : b.index_scans) {  // class index + first interval -> offsets of the scan's slices
        const ScanClass &cl = b.classes[(size_t)is.off_arr];
        const uint64_t first = is.end_arr * sizeof(uint64_t);
        is.off_arr = cl.dev_intervals + first;
        is.end_arr = cl.dev_interval_end + first;
        is.clean_arr = cl.dev_clean_off + first;
    }
    b.input_bytes = cur;
}

// pinned staging of the input buffer + device memory; returns 0 or the status the batch fails with
static int stage_and_allocate(b200jpg_batch &b, const Codestreams &cs, const std::vector<uint64_t> &byte_off) {
    b200jpg_ctx *ctx = b.ctx;
    cudaError_t ce;
    b.h_input = (uint8_t *)ctx->get(0, b.input_bytes, &ce);
    if (ce != cudaSuccess) return ctx->fail(B200JPG_ERR_OUT_OF_MEMORY, std::string("pinned staging allocation failed: ") + cudaGetErrorString(ce));
    for_frames(b.n, 8, [&](int i) {
        if (b.parse_status[i] != 0) return;
        uint8_t *dst = b.h_input + byte_off[i];
        memcpy(dst, cs.data[i], cs.len[i]);
        // sentinel: a damaged segment must still meet a marker before it leaves its codestream
        uint64_t pad_end = align_up(byte_off[i] + cs.len[i] + 32, 16);
        memset(dst + cs.len[i], 0, pad_end - (byte_off[i] + cs.len[i]));
        dst[cs.len[i]] = 0xff;
        dst[cs.len[i] + 1] = 0xd9;
    });
    // tail of the codestream region (after the last frame) is zero + a final sentinel
    {
        uint64_t last_end = 0;
        for (int i = 0; i < b.n; i++)
            if (b.parse_status[i] == 0) last_end = align_up(byte_off[i] + cs.len[i] + 32, 16);
        memset(b.h_input + last_end, 0, b.bytes_region - last_end);
        b.h_input[last_end] = 0xff;
        b.h_input[last_end + 1] = 0xd9;
    }
    for (size_t t = 0; t < b.table_sets.size(); t++)
        memcpy(b.h_input + b.dev_tables[t], b.table_sets[t].blob.data(), b.table_sets[t].blob.size());
    for (auto &cl : b.classes) {
        memcpy(b.h_input + cl.dev_scans, cl.scans.data(), cl.scans.size() * sizeof(ClassScan));
        memcpy(b.h_input + cl.dev_intervals, cl.interval_off.data(), cl.interval_off.size() * sizeof(uint64_t));
        memcpy(b.h_input + cl.dev_interval_end, cl.interval_end.data(), cl.interval_end.size() * sizeof(uint64_t));
        memcpy(b.h_input + cl.dev_clean_off, cl.clean_off.data(), cl.clean_off.size() * sizeof(uint64_t));
    }
    for (auto &g : b.groups) memcpy(b.h_input + g.dev_frames, g.frames.data(), g.frames.size() * sizeof(FrameRecon));
    if (!b.index_scans.empty()) memcpy(b.h_input + b.dev_index_scans, b.index_scans.data(), b.index_scans.size() * sizeof(IndexScan));
    if (!b.prog_frames.empty()) memcpy(b.h_input + b.dev_prog_frames, b.prog_frames.data(), b.prog_frames.size() * sizeof(ProgFrame));
    if (!b.rs_frames.empty()) memcpy(b.h_input + b.dev_rs_frames, b.rs_frames.data(), b.rs_frames.size() * sizeof(ResampleFrame));
    for (size_t r = 0; r < b.rs_frames.size(); r++) {
        const ResampleFrame &f = b.rs_frames[r];
        const uint64_t at[4] = {f.h_bounds, f.h_coef, f.v_bounds, f.v_coef};
        for (int t = 0; t < 4; t++) {
            const std::vector<int32_t> &v = b.rs_tables[r][t];
            const uint64_t bytes = v.size() * sizeof(int32_t);
            if (bytes) memcpy(b.h_input + at[t], v.data(), bytes);
            memset(b.h_input + at[t] + bytes, 0, align_up(bytes, 16) - bytes);
        }
    }

    b.sz_ilen = sizeof(uint32_t) * (size_t)std::max<uint64_t>(b.n_intervals, 1);
    b.sz_status = sizeof(uint32_t) * (5 * (size_t)b.n + 1);  // status words, wide flags, narrow flags, narrow list, index status
    b.d_input = (uint8_t *)ctx->get(1, b.input_bytes, &ce);
    if (ce == cudaSuccess && b.coef_elems) b.d_coef = (int16_t *)ctx->get(1, b.coef_elems * sizeof(int16_t), &ce);
    if (ce == cudaSuccess && b.sample_elems) b.d_samples = (int32_t *)ctx->get(1, b.sample_elems * sizeof(int32_t), &ce);
    // the int16 planes serve the Tiled path only, which downscaled batches never take
    if (ce == cudaSuccess && b.sample_elems && downscale_of(b.flags) == 1) b.d_samples16 = (int16_t *)ctx->get(1, b.sample_elems * sizeof(int16_t), &ce);
    if (ce == cudaSuccess && b.plane8_bytes) b.d_planes8 = (uint8_t *)ctx->get(1, b.plane8_bytes, &ce);
    if (ce == cudaSuccess) b.d_clean = (uint8_t *)ctx->get(1, b.clean_bytes, &ce);
    if (ce == cudaSuccess) b.d_interval_len = (uint32_t *)ctx->get(1, b.sz_ilen, &ce);
    b.sz_overrun = sizeof(uint32_t) * (size_t)(b.n_intervals + b.classes.size() + 1);
    if (ce == cudaSuccess) b.d_overrun = (uint32_t *)ctx->get(1, b.sz_overrun, &ce);
    if (ce == cudaSuccess) b.d_status = (uint32_t *)ctx->get(1, b.sz_status, &ce);
    if (ce == cudaSuccess && !b.pf_groups.empty()) b.d_dcplane = (int16_t *)ctx->get(1, b.coef_elems / 64 * sizeof(int16_t), &ce);
    if (ce == cudaSuccess && b.n_spec) {
        b.sz_spec = (size_t)align_up(b.n_spec, 4) * (sizeof(SpecSegment) + 8 + 8 + 4 + 16 + sizeof(SpecLog)) + 256;
        b.d_spec = (uint8_t *)ctx->get(1, b.sz_spec, &ce);
    }
    if (ce == cudaSuccess && b.scratch_bytes) b.d_scratch = (uint8_t *)ctx->get(1, b.scratch_bytes, &ce);
    if (ce == cudaSuccess && b.inter_bytes) b.d_inter = (uint8_t *)ctx->get(1, b.inter_bytes, &ce);
    if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&b.ev_last, cudaEventDisableTiming);
    if (ce != cudaSuccess) return ctx->fail(B200JPG_ERR_OUT_OF_MEMORY, std::string("device allocation failed: ") + cudaGetErrorString(ce));
    b.h_status.assign(b.n, 0);
    return B200JPG_OK;
}

// The live frames' rectangles C (a failed frame's request is ignored): b200jpg_batch_create_crop's (nullptr: none), each checked
// against the frame's uncropped output extent, else the whole output for a frame with a target size, so that the reconstruction
// writes C through the cropped path, and for every frame under B200JPG_FLAG_LIBJPEG_TURBO, so that turbo_generic_kernel needs only
// the clipped strided store kinds, whatever the destination. A cropped frame is described. Returns 0 or the status the call fails with.
static int admit_crops(b200jpg_batch &b, const b200jpg_rect *rects) {
    for (int i = 0; i < b.n_user; i++) {
        FramePlan &p = b.plan[i];
        b200jpg_rect r = rects ? rects[i] : b200jpg_rect{0, 0, 0, 0};
        const bool whole = !size_empty(p.target) || (b.flags & B200JPG_FLAG_LIBJPEG_TURBO);
        if (b.parse_status[i] != 0 || (rect_empty(r) && !whole)) continue;
        const Extent e = out_extent(b.frames[i].info, 0, b.flags, p);
        if (rect_empty(r)) r = b200jpg_rect{0, 0, (uint32_t)e.w, (uint32_t)e.h};
        if (r.width == 0 || r.height == 0 || (uint64_t)r.x + r.width > e.w || (uint64_t)r.y + r.height > e.h)
            return b.ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "frame " + std::to_string(i) + ": crop rectangle (" + std::to_string(r.x) + ", " +
                                                                  std::to_string(r.y) + ", " + std::to_string(r.width) + ", " + std::to_string(r.height) +
                                                                  ") is empty or leaves the " + std::to_string(e.w) + " x " + std::to_string(e.h) + " output");
        // a flip without a size is in the orientation (frame_plan): r, given in the unflipped image, as a rectangle of the flipped one
        p.crop = size_empty(p.target) ? flip_rect(r, p.flip, e.w, e.h) : r;
        p.cropped = p.described = true;
    }
    return B200JPG_OK;
}

// b200jpg_batch_create_resize's sizes (in the records since batch creation began: attach_residuals reads them), for the live frames
// (a failed frame's is ignored); returns 0 or the status the call fails with (a size whose bitmaps could never be allocated)
static int admit_sizes(b200jpg_batch &b) {
    for (int i = 0; i < b.n_user; i++) {
        FramePlan &p = b.plan[i];
        const b200jpg_size &s = p.target;
        if (b.parse_status[i] != 0 || size_empty(s)) continue;
        if (s.width > (1u << 24) || s.height > (1u << 24) || (uint64_t)s.width * s.height * p.out_ncomp > (1ull << 34))
            return b.ctx->fail(B200JPG_ERR_OUT_OF_MEMORY, "frame " + std::to_string(i) + ": target size " + std::to_string(s.width) + " x " +
                                                              std::to_string(s.height) + " is too large to allocate");
        p.resized = true;
    }
    return B200JPG_OK;
}

// b200jpg_batch_create_draft's requests (nullptr: none): every caller's frame's factor k, B200JPG_FLAG_DOWNSCALE_k or, for a live
// frame with a request, Pillow's draft scale (a failed frame's request is ignored)
static void admit_drafts(b200jpg_batch &b, const b200jpg_size *drafts) {
    for (int i = 0; i < b.n_user; i++) {
        b.plan[i].k = downscale_of(b.flags);
        if (drafts && b.parse_status[i] == 0 && !size_empty(drafts[i])) b.plan[i].k = draft_scale_of(b.frames[i].info, drafts[i].width, drafts[i].height);
    }
}

// Pillow's _filters_support
static double filter_support(int resample) {
    switch (resample) {
    case B200JPG_RESAMPLE_BOX: return 0.5;
    case B200JPG_RESAMPLE_BICUBIC: return 2.0;
    case B200JPG_RESAMPLE_LANCZOS: return 3.0;
    default: return 1.0;  // bilinear, hamming
    }
}

// Image.resize's reduce step for resized frame i (DESIGN §19), in double as Pillow's Python computes it: the factors, the reduce
// box rb in C (x0, y0, x1, y1; Image._get_safe_box) and the box the resampler then takes, in the reduced image's coordinates (C's
// when the frame does not reduce). C is the frame's rectangle FramePlan::crop, untrimmed.
struct ReducePlan {
    uint64_t fx = 1, fy = 1;
    int64_t rb[4] = {0, 0, 0, 0};
    double box[4];
};
static ReducePlan reduce_plan(const b200jpg_batch &b, int i) {
    const b200jpg_rect &c = b.plan[i].crop;
    const b200jpg_size &t = b.plan[i].target;
    ReducePlan p;
    const b200jpg_box &bx = b.plan[i].box;
    const double box[4] = {bx.x0, bx.y0, bx.x1, bx.y1}, whole[4] = {0.0, 0.0, (double)c.width, (double)c.height};
    memcpy(p.box, box_empty(bx) ? whole : box, sizeof(p.box));
    if (b.gap <= 0.0) return p;
    p.fx = std::max<uint64_t>(1, (uint64_t)((p.box[2] - p.box[0]) / t.width / b.gap));  // int(...) or 1
    p.fy = std::max<uint64_t>(1, (uint64_t)((p.box[3] - p.box[1]) / t.height / b.gap));
    if (p.fx == 1 && p.fy == 1) return p;
    const double support = filter_support(b.resample) - 0.5;
    const double sx = support * ((p.box[2] - p.box[0]) / t.width), sy = support * ((p.box[3] - p.box[1]) / t.height);
    p.rb[0] = std::max<int64_t>(0, (int64_t)(p.box[0] - sx));
    p.rb[1] = std::max<int64_t>(0, (int64_t)(p.box[1] - sy));
    p.rb[2] = std::min<int64_t>(c.width, (int64_t)std::ceil(p.box[2] + sx));
    p.rb[3] = std::min<int64_t>(c.height, (int64_t)std::ceil(p.box[3] + sy));
    const double nb[4] = {(p.box[0] - p.rb[0]) / p.fx, (p.box[1] - p.rb[1]) / p.fy, (p.box[2] - p.rb[0]) / p.fx, (p.box[3] - p.rb[1]) / p.fy};
    memcpy(p.box, nb, sizeof(p.box));
    return p;
}

// Which rule of DESIGN §20 cv2.resize applies to resized frame i (C, the frame's untrimmed rectangle, to its target), as OpenCV
// decides it: 0 for the copy (same size), 1 for INTER_LINEAR; for INTER_AREA 2 where both axes shrink by integer factors
// (|scale - round(scale)| < DBL_EPSILON), 3 where both scales are >= 1 otherwise, 4 where either axis grows.
struct CvPlan {
    int rule = 0;
    uint64_t fx = 1, fy = 1;  // rule 2's factors
};
static CvPlan cv_plan(const b200jpg_batch &b, int i) {
    const b200jpg_rect &c = b.plan[i].crop;
    const b200jpg_size &t = b.plan[i].target;
    CvPlan p;
    if (c.width == t.width && c.height == t.height) return p;
    if (b.resample == B200JPG_RESAMPLE_CV_LINEAR) return p.rule = 1, p;
    const double sx = 1.0 / ((double)t.width / c.width), sy = 1.0 / ((double)t.height / c.height);
    if (sx < 1.0 || sy < 1.0) return p.rule = 4, p;
    const double ix = std::nearbyint(sx), iy = std::nearbyint(sy);
    if (std::fabs(sx - ix) < DBL_EPSILON && std::fabs(sy - iy) < DBL_EPSILON) return p.rule = 2, p.fx = (uint64_t)ix, p.fy = (uint64_t)iy, p;
    return p.rule = 3, p;
}

// b200jpg_batch_create_resample's boxes and windows (nullptr: none), checked for the live frames (a failed frame's are ignored)
// against C (the frame's rectangle, set by admit_crops) and the target size; a frame without a target size refuses both (a window
// replaces the frame's output extent: out_extent). Under OpenCV's filters a box is refused and so are rule 2's blocks whose int
// sums could overflow (DESIGN §20). Returns 0 or the status the call fails with.
static int admit_boxes(b200jpg_batch &b, const b200jpg_box *boxes, const b200jpg_rect *windows) {
    for (int i = 0; i < b.n_user; i++) {
        if (b.parse_status[i] != 0) continue;
        FramePlan &p = b.plan[i];
        const b200jpg_box bx = boxes ? boxes[i] : b200jpg_box{0, 0, 0, 0};
        const b200jpg_rect wn = windows ? windows[i] : b200jpg_rect{0, 0, 0, 0};
        const std::string at = "frame " + std::to_string(i) + ": ";
        if (!box_empty(bx) || !rect_empty(wn)) {
            if (!p.resized) return b.ctx->fail(B200JPG_ERR_INVALID_PARAMETER, at + "a box or window needs a target size");
            const b200jpg_rect &c = p.crop;
            const b200jpg_size &t = p.target;
            if (!box_empty(bx) && resample_cv(b.resample))
                return b.ctx->fail(B200JPG_ERR_INVALID_PARAMETER, at + "OpenCV's resize takes no source box");
            if (!box_empty(bx)) {
                const std::string desc = "box (" + std::to_string(bx.x0) + ", " + std::to_string(bx.y0) + ", " + std::to_string(bx.x1) + ", " +
                                         std::to_string(bx.y1) + ")";
                if (!std::isfinite(bx.x0) || !std::isfinite(bx.y0) || !std::isfinite(bx.x1) || !std::isfinite(bx.y1))
                    return b.ctx->fail(B200JPG_ERR_INVALID_PARAMETER, at + desc + " is not finite");
                if (bx.x0 < 0.0 || bx.y0 < 0.0) return b.ctx->fail(B200JPG_ERR_INVALID_PARAMETER, at + desc + " has a negative offset");
                if (bx.x1 > c.width || bx.y1 > c.height)
                    return b.ctx->fail(B200JPG_ERR_INVALID_PARAMETER,
                                       at + desc + " leaves the " + std::to_string(c.width) + " x " + std::to_string(c.height) + " image");
                if (bx.x1 < bx.x0 || bx.y1 < bx.y0) return b.ctx->fail(B200JPG_ERR_INVALID_PARAMETER, at + desc + " has a negative extent");
            }
            if (!rect_empty(wn) && (wn.width == 0 || wn.height == 0 || (uint64_t)wn.x + wn.width > t.width || (uint64_t)wn.y + wn.height > t.height))
                return b.ctx->fail(B200JPG_ERR_INVALID_PARAMETER, at + "window (" + std::to_string(wn.x) + ", " + std::to_string(wn.y) + ", " +
                                                                      std::to_string(wn.width) + ", " + std::to_string(wn.height) +
                                                                      ") is empty or leaves the " + std::to_string(t.width) + " x " +
                                                                      std::to_string(t.height) + " image");
            p.box = bx;
            p.window = wn;
        }
        if (p.resized && resample_cv(b.resample)) {  // rule 2's int sums: 255 fx fy below 2^31
            const CvPlan cp = cv_plan(b, i);
            if (cp.rule == 2 && 255ull * cp.fx * cp.fy >= (1ull << 31))
                return b.ctx->fail(B200JPG_ERR_NOT_IMPLEMENTED, at + "area blocks of " + std::to_string(cp.fx) + " x " + std::to_string(cp.fy) +
                                                                    " pixels overflow OpenCV's int sums");
        }
        if (!p.resized || b.gap <= 0.0) continue;
        const ReducePlan rp = reduce_plan(b, i);
        if (rp.fx * rp.fy >= (1ull << 24))
            return b.ctx->fail(B200JPG_ERR_NOT_IMPLEMENTED, at + "reduce factors " + std::to_string(rp.fx) + " x " + std::to_string(rp.fy) +
                                                                " reach 2^24 pixels per block");
        if ((rp.fx > 1 || rp.fy > 1) && (rp.rb[2] <= rp.rb[0] || rp.rb[3] <= rp.rb[1]))
            return b.ctx->fail(B200JPG_ERR_INVALID_PARAMETER, at + "the reduce box of the source box is empty");
    }
    return B200JPG_OK;
}

// One axis of resized frame i: the table of the source's `in` samples for `out` outputs (box: Pillow's floats, nullptr for the
// default box), restricted to the window's outputs [w0, w0 + wn), or none when Pillow does not resample the axis. Returns the
// source range [lo, hi) the window reads, the tables rebased to lo.
static void plan_axis(uint32_t in, const float *box, uint32_t out, uint32_t w0, uint32_t wn, int resample, bool pass,
                      std::vector<int32_t> &bounds, std::vector<int32_t> &coef, uint32_t &ksize, uint32_t &lo, uint32_t &hi) {
    if (!pass) {  // the window's own samples (out == in)
        lo = w0, hi = w0 + wn;
        return;
    }
    resample_coefficients(in, box, out, resample, bounds, coef, ksize);  // (the arguments are valid: the call cannot fail)
    if (w0 != 0 || wn != out) {
        bounds.erase(bounds.begin() + 2 * ((size_t)w0 + wn), bounds.end());
        bounds.erase(bounds.begin(), bounds.begin() + 2 * (size_t)w0);
        coef.erase(coef.begin() + ((size_t)w0 + wn) * ksize, coef.end());
        coef.erase(coef.begin(), coef.begin() + (size_t)w0 * ksize);
    }
    lo = in, hi = 0;
    for (uint32_t j = 0; j < wn; j++)
        if (bounds[2 * j + 1] > 0) lo = std::min<uint32_t>(lo, bounds[2 * j]), hi = std::max<uint32_t>(hi, bounds[2 * j] + bounds[2 * j + 1]);
    if (lo >= hi) lo = 0, hi = 1;  // no output reads a sample (a zero-width box at the edge): one sample stays
    for (uint32_t j = 0; j < wn; j++) bounds[2 * j] = bounds[2 * j + 1] > 0 ? bounds[2 * j] - (int32_t)lo : 0;
}

// One axis of a frame under OpenCV's rules 1, 3 and 4 (DESIGN §20): the table of `table` (b200jpg_resample_coefficients' encoding;
// `pairs`: the two-tap tables of rules 1 / 4) restricted to the window's outputs [w0, w0 + wn), rebased to the source range [lo, hi)
// it reads.
static void plan_cv_axis(uint32_t in, uint32_t out, uint32_t w0, uint32_t wn, int table, bool pairs, std::vector<int32_t> &bounds,
                         std::vector<int32_t> &coef, uint32_t &ksize, uint32_t &lo, uint32_t &hi) {
    cv_resample_coefficients(in, out, table, bounds, coef, ksize);  // (the arguments are valid: the call cannot fail)
    if (w0 != 0 || wn != out) {
        bounds.erase(bounds.begin() + 2 * ((size_t)w0 + wn), bounds.end());
        bounds.erase(bounds.begin(), bounds.begin() + 2 * (size_t)w0);
        coef.erase(coef.begin() + ((size_t)w0 + wn) * ksize, coef.end());
        coef.erase(coef.begin(), coef.begin() + (size_t)w0 * ksize);
    }
    lo = in, hi = 0;
    for (uint32_t j = 0; j < wn; j++) {
        const uint32_t a = bounds[2 * j], e = pairs ? bounds[2 * j + 1] + 1 : a + bounds[2 * j + 1];
        if (e > a) lo = std::min(lo, a), hi = std::max(hi, e);
    }
    if (lo >= hi) lo = 0, hi = 1;
    for (uint32_t j = 0; j < wn; j++) {
        bounds[2 * j] = std::max<int32_t>(bounds[2 * j] - (int32_t)lo, 0);
        if (pairs) bounds[2 * j + 1] -= (int32_t)lo;
    }
}

// A resized frame under OpenCV's filters: the blocks of rule 2 (and the copy) read C from the window's first block on; rules 1, 3
// and 4 run the two passes over what their tables read.
static void plan_cv_frame(const b200jpg_batch &b, int i, ResampleFrame &f, std::array<std::vector<int32_t>, 4> &t, b200jpg_rect &c) {
    const CvPlan cp = cv_plan(b, i);
    const b200jpg_size &s = b.plan[i].target;
    const b200jpg_rect &wn = b.plan[i].window;
    const uint32_t wx = rect_empty(wn) ? 0 : wn.x, wy = rect_empty(wn) ? 0 : wn.y;
    if (cp.rule == 0 || cp.rule == 2) {
        f.fx = (uint32_t)cp.fx, f.fy = (uint32_t)cp.fy;
        c.x += wx * f.fx, c.y += wy * f.fy, c.width = f.tw * f.fx, c.height = f.th * f.fy;
        f.w = c.width, f.h = c.height;
        return;
    }
    f.pass = kPassH | kPassV | (cp.rule == 3 ? kPassArea : 0u);
    const int table = b.resample | (cp.rule == 4 ? B200JPG_CV_TABLE_LINEAR : 0);
    uint32_t x0, x1, y0, y1;
    plan_cv_axis(c.width, s.width, wx, f.tw, table, cp.rule != 3, t[0], t[1], f.h_ksize, x0, x1);
    plan_cv_axis(c.height, s.height, wy, f.th, table | B200JPG_CV_TABLE_VERTICAL, cp.rule != 3, t[2], t[3], f.v_ksize, y0, y1);
    f.w = x1 - x0, f.h = y1 - y0;
    c.x += x0, c.y += y0, c.width = f.w, c.height = f.h;
}

// The resample descriptors and tables of the resized frames (tables built on host threads, one frame each) and the layout of the
// scratch (C: c_h rows of align16(c_w * ncomp) bytes per frame, then R where the frame reduces) and of the intermediate (rows y0 ..
// y1 - 1 of tw * ncomp bytes, for frames with a horizontal pass). The grey frames of B200JPG_FLAG_OUTPUT_RGB come last, with one
// channel: the vertical pass replicates it. Each frame's rectangle shrinks to the part of C its tables (or its reduce box) read,
// which is all of C without a box, a window and a reduce (DESIGN §19): the reconstruction covers no more.
static void plan_resample(b200jpg_batch &b) {
    std::vector<int> rs_user;  // [resized] caller frame
    for (int rgb = 0; rgb < 2; rgb++) {
        for (int i = 0; i < b.n_user; i++)
            if (b.parse_status[i] == 0 && b.plan[i].resized && (b.plan[i].mode == OutMode::Replicate) == (rgb == 1)) {
                b.plan[i].rs = (int)rs_user.size();
                rs_user.push_back(i);
            }
        if (rgb == 0) b.rs_plain = (uint32_t)rs_user.size();
    }
    const int nr = (int)rs_user.size();
    b.rs_frames.assign(nr, ResampleFrame{});
    b.rs_tables.assign(nr, {});
    for_frames(nr, 16, [&](int r) {
        const int i = rs_user[r];
        FramePlan &plan = b.plan[i];  // C has the components the reconstruction stores
        b200jpg_rect &c = plan.crop;  // C, trimmed below to what the resize reads
        const b200jpg_size &s = plan.target;
        const b200jpg_rect &wn = plan.window;
        ResampleFrame &f = b.rs_frames[r];
        auto &t = b.rs_tables[r];
        f.ncomp = plan.mode == OutMode::Replicate ? plan.ncomp : plan.out_ncomp;
        f.plane = (uint32_t)(b.n + r);
        if (resample_cv(b.resample)) {  // (DESIGN §20)
            f.tw = rect_empty(wn) ? s.width : wn.width, f.th = rect_empty(wn) ? s.height : wn.height;
            f.fx = f.fy = 1;
            plan_cv_frame(b, i, f, t, c);
            f.c_w = c.width, f.c_h = c.height;
            f.c_pitch = f.src_pitch = (uint32_t)align_up((uint64_t)f.w * f.ncomp, 16);
            f.y0 = 0, f.y1 = f.h;
            if (f.src_pitch <= kResampleRowSmem) f.stage |= kStageRow;
            if ((f.pass & kPassH) && align_up(t[1].size() * sizeof(int32_t), 16) <= kResampleCoefSmem) f.stage |= kStageCoef;
            return;
        }
        const ReducePlan rp = reduce_plan(b, i);
        const bool reduces = rp.fx > 1 || rp.fy > 1;
        f.fx = (uint32_t)rp.fx, f.fy = (uint32_t)rp.fy;
        // the source S: R, (rb.x1 - rb.x0) / fx x (rb.y1 - rb.y0) / fy rounded up, or C
        const uint32_t sw = reduces ? (uint32_t)((rp.rb[2] - rp.rb[0] + rp.fx - 1) / rp.fx) : c.width;
        const uint32_t sh = reduces ? (uint32_t)((rp.rb[3] - rp.rb[1] + rp.fy - 1) / rp.fy) : c.height;
        const float fb[4] = {(float)rp.box[0], (float)rp.box[1], (float)rp.box[2], (float)rp.box[3]};  // Pillow's "(ffff)"
        const bool plain = !reduces && box_empty(plan.box);  // DESIGN §13's tables, computed as they always were
        f.pass = (s.width != sw || fb[0] != 0.0f || fb[2] != (float)s.width ? kPassH : 0u) |
                 (s.height != sh || fb[1] != 0.0f || fb[3] != (float)s.height ? kPassV : 0u);
        f.tw = rect_empty(wn) ? s.width : wn.width, f.th = rect_empty(wn) ? s.height : wn.height;
        const float fbh[2] = {fb[0], fb[2]}, fbv[2] = {fb[1], fb[3]};
        uint32_t x0, x1, y0, y1;  // the part of S the window reads
        plan_axis(sw, plain ? nullptr : fbh, s.width, wn.x, f.tw, b.resample, f.pass & kPassH, t[0], t[1], f.h_ksize, x0, x1);
        plan_axis(sh, plain ? nullptr : fbv, s.height, wn.y, f.th, b.resample, f.pass & kPassV, t[2], t[3], f.v_ksize, y0, y1);
        f.w = x1 - x0, f.h = y1 - y0;
        f.src_pitch = (uint32_t)align_up((uint64_t)f.w * f.ncomp, 16);
        if (reduces) {  // R's blocks x0 .. x1 - 1, y0 .. y1 - 1: the pixels of C they cover (the last ones partial only at rb's edges)
            const uint64_t cx = rp.rb[0] + (uint64_t)x0 * rp.fx, cy = rp.rb[1] + (uint64_t)y0 * rp.fy;
            c.x += (uint32_t)cx, c.y += (uint32_t)cy;
            c.width = (uint32_t)(std::min<uint64_t>(rp.rb[2], rp.rb[0] + (uint64_t)x1 * rp.fx) - cx);
            c.height = (uint32_t)(std::min<uint64_t>(rp.rb[3], rp.rb[1] + (uint64_t)y1 * rp.fy) - cy);
        } else {
            c.x += x0, c.y += y0, c.width = f.w, c.height = f.h;
        }
        f.c_w = c.width, f.c_h = c.height;
        f.c_pitch = (uint32_t)align_up((uint64_t)f.c_w * f.ncomp, 16);
        f.y0 = 0, f.y1 = f.h;
        if (f.src_pitch <= kResampleRowSmem) f.stage |= kStageRow;
        if ((f.pass & kPassH) && align_up(t[1].size() * sizeof(int32_t), 16) <= kResampleCoefSmem) f.stage |= kStageCoef;
    });
    const bool cv = resample_cv(b.resample);
    for (ResampleFrame &f : b.rs_frames) {
        f.c_src = f.src = b.scratch_bytes;
        b.scratch_bytes = align_up(b.scratch_bytes + (uint64_t)f.c_pitch * f.c_h, 256);
        if (cv) b.rs_cv_kinds |= !f.pass ? kCvBlocks : (f.pass & kPassArea) ? kCvArea : kCvLinear;
        if (!cv && (f.fx > 1 || f.fy > 1)) {  // R behind C
            f.src = b.scratch_bytes;
            b.scratch_bytes = align_up(b.scratch_bytes + (uint64_t)f.src_pitch * f.h, 256);
            b.rs_max_reduce_rows = std::max(b.rs_max_reduce_rows, f.h);
        }
        if (f.pass & kPassH) {
            f.inter = b.inter_bytes;
            b.inter_bytes = align_up(b.inter_bytes + (uint64_t)(f.y1 - f.y0) * f.tw * f.ncomp * (cv ? 4 : 1), 256);  // (cv: int32 / float)
            b.rs_max_rows = std::max(b.rs_max_rows, f.y1 - f.y0);
        }
        b.rs_max_pixels = std::max(b.rs_max_pixels, (uint64_t)f.tw * f.th);
    }
}

static int batch_create_impl(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad, unsigned flags,
                             const b200jpg_size *drafts, const b200jpg_rect *rects, const b200jpg_size *sizes, const b200jpg_box *boxes,
                             const b200jpg_rect *windows, int resample, double reducing_gap, const uint8_t *flips, b200jpg_batch **out) {
    NvtxRange nvtx("b200jpg batch_create: parse + pack");
    if (!out || !frames || !lens || n <= 0) return ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "invalid batch arguments");
    *out = nullptr;
    bool any_flip = false;
    for (int i = 0; flips && i < n; i++) {
        if (flips[i] & ~(B200JPG_FLIP_H | B200JPG_FLIP_V))
            return ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "frame " + std::to_string(i) + ": flip " + std::to_string(flips[i]) +
                                                                " has a bit other than B200JPG_FLIP_H and B200JPG_FLIP_V");
        any_flip = any_flip || flips[i] != 0;
    }
    if (!any_flip) flips = nullptr;  // all zero: exactly the batch of b200jpg_batch_create_resample
    if (std::isnan(reducing_gap) || (reducing_gap > 0.0 && reducing_gap < 1.0))
        return ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "reducing_gap " + std::to_string(reducing_gap) + " is NaN or below 1.0");
    bool any_box = false;
    for (int i = 0; i < n; i++) any_box = any_box || (boxes && !box_empty(boxes[i])) || (windows && !rect_empty(windows[i]));
    if (!any_box) boxes = nullptr, windows = nullptr;  // all zero: exactly the batch of b200jpg_batch_create_draft
    bool any_draft = false;
    for (int i = 0; drafts && i < n; i++) {
        if ((drafts[i].width == 0) != (drafts[i].height == 0))
            return ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "frame " + std::to_string(i) + ": draft size " + std::to_string(drafts[i].width) + " x " +
                                                                std::to_string(drafts[i].height) + " has exactly one zero side");
        any_draft = any_draft || !size_empty(drafts[i]);
    }
    if (!any_draft) drafts = nullptr;  // all {0, 0}: exactly the batch of b200jpg_batch_create_resize
    if (drafts && !(flags & B200JPG_FLAG_LIBJPEG_TURBO))
        return ctx->fail(B200JPG_ERR_NOT_IMPLEMENTED, "a draft size needs B200JPG_FLAG_LIBJPEG_TURBO (libjpeg-turbo's reduced decode)");
    bool any_crop = false;
    for (int i = 0; rects && i < n; i++) any_crop = any_crop || !rect_empty(rects[i]);
    if (!any_crop) rects = nullptr;  // all {0, 0, 0, 0}: exactly the batch of b200jpg_batch_create_ex
    bool any_size = false;
    for (int i = 0; sizes && i < n; i++) {
        if ((sizes[i].width == 0) != (sizes[i].height == 0))
            return ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "frame " + std::to_string(i) + ": target size " + std::to_string(sizes[i].width) + " x " +
                                                                std::to_string(sizes[i].height) + " has exactly one zero side");
        if (!size_empty(sizes[i]) && !resample_known(resample) && !resample_cv(resample))
            return ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "frame " + std::to_string(i) + ": unknown resample filter " + std::to_string(resample));
        if (!size_empty(sizes[i]) && resample_cv(resample) && reducing_gap > 0.0)
            return ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "frame " + std::to_string(i) + ": OpenCV's resize takes no reducing_gap");
        any_size = any_size || !size_empty(sizes[i]);
    }
    if (!any_size) sizes = nullptr;  // all {0, 0}: exactly the batch of b200jpg_batch_create_crop
    if (rects && (flags & B200JPG_FLAG_NO_UPSAMPLE))
        return ctx->fail(B200JPG_ERR_NOT_IMPLEMENTED, "crop rectangles are not supported with B200JPG_FLAG_NO_UPSAMPLE");
    if (sizes && (flags & B200JPG_FLAG_NO_UPSAMPLE))
        return ctx->fail(B200JPG_ERR_NOT_IMPLEMENTED, "target sizes are not supported with B200JPG_FLAG_NO_UPSAMPLE");
    if ((flags & kOutputModes) == kOutputModes)
        return ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "B200JPG_FLAG_OUTPUT_RGB and B200JPG_FLAG_OUTPUT_L exclude each other");
    if ((flags & kOutputModes) && (flags & B200JPG_FLAG_NO_UPSAMPLE))
        return ctx->fail(B200JPG_ERR_NOT_IMPLEMENTED, "an output mode is not supported with B200JPG_FLAG_NO_UPSAMPLE");
    if ((flags & kOutputModes) && (flags & B200JPG_FLAG_NO_COLOR_TRANSFORM))
        return ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "an output mode needs the colour transformation (no B200JPG_FLAG_NO_COLOR_TRANSFORM)");
    if ((flags & B200JPG_FLAG_LIBJPEG_TURBO) && (flags & (B200JPG_FLAG_DOWNSCALE_MASK | B200JPG_FLAG_NO_UPSAMPLE)))
        return ctx->fail(B200JPG_ERR_NOT_IMPLEMENTED, "B200JPG_FLAG_LIBJPEG_TURBO is not supported with B200JPG_FLAG_DOWNSCALE_k or B200JPG_FLAG_NO_UPSAMPLE");
    cudaError_t ce = cudaSetDevice(ctx->device);
    if (ce != cudaSuccess) return ctx->fail_cuda(ce, "cudaSetDevice");

    std::unique_ptr<b200jpg_batch, void (*)(b200jpg_batch *)> bp(new b200jpg_batch(), b200jpg_batch_destroy);  // a failed plan frees what it holds
    b200jpg_batch &b = *bp;
    b.ctx = ctx;
    b.n = b.n_user = n;
    b.flags = flags;
    b.plan.assign(n, FramePlan{});
    for (int i = 0; sizes && i < n; i++) b.plan[i].target = sizes[i];  // (attach_residuals refuses 12-bit frames with a size)
    for (int i = 0; flips && i < n; i++) b.plan[i].flip = flips[i];    // (read by frame_plan, admit_crops and the descriptor table)
    if (sizes) b.resample = resample, b.gap = reducing_gap;  // (gap <= 0: None)
    Codestreams cs;
    cs.data.assign(frames, frames + n);
    cs.len.assign(lens, lens + n);
    cs.err.resize(n);
    // Interleaved scans with restart markers get their restart index on the device (8f1); B200JPG_HOST_INDEX=1 keeps the memchr
    // pass over every entropy coded byte on the host for all of them.
    const bool device_index = getenv("B200JPG_HOST_INDEX") == nullptr;
    parse_frames(b, cs, device_index);
    attach_residuals(b, cs, device_index);
    std::vector<std::vector<TableSet>> frame_tables;
    if (int rc = admit_frames(b, cs, tolerate_bad != 0, frame_tables)) return rc;
    admit_drafts(b, drafts);
    for (int i = 0; i < n; i++)
        if (b.parse_status[i] == 0) frame_plan(b, i);
    if (int rc = admit_crops(b, rects)) return rc;
    if (int rc = admit_sizes(b)) return rc;
    if (boxes || windows || b.gap > 0.0 || resample_cv(b.resample))
        if (int rc = admit_boxes(b, boxes, windows)) return rc;
    plan_resample(b);  // (before the reconstruction groups: it trims the rectangles of resized frames)
    for (int i = n; i < b.n; i++)  // JPEG XT residual codestreams: their frames' records, their own components
        if (b.parse_status[i] == 0) b.plan[i] = b.plan[b.xt_parent[i]], b.plan[i].ncomp = b.frames[i].info.ncomp;
    const std::vector<uint64_t> byte_off = lay_out_codestreams(b, cs.len);
    const std::vector<std::array<uint64_t, 4>> sample_base = lay_out_planes(b);
    form_scan_classes(b, frame_tables, byte_off);
    form_progressive_groups(b);
    lay_out_unstuffed(b);
    form_recon_groups(b, sample_base);
    lay_out_descriptors(b);
    if (int rc = stage_and_allocate(b, cs, byte_off)) return rc;
    *out = bp.release();
    return B200JPG_OK;
}

int b200jpg_batch_create(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad,
                         b200jpg_batch **out) {
    return b200jpg_batch_create_ex(ctx, frames, lens, n, tolerate_bad, 0u, out);
}

int b200jpg_batch_create_ex(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad, unsigned flags,
                            b200jpg_batch **out) {
    return b200jpg_batch_create_crop(ctx, frames, lens, n, tolerate_bad, flags, nullptr, out);
}

int b200jpg_batch_create_crop(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad, unsigned flags,
                              const b200jpg_rect *rects, b200jpg_batch **out) {
    return b200jpg_batch_create_resize(ctx, frames, lens, n, tolerate_bad, flags, rects, nullptr, 0, out);
}

int b200jpg_batch_create_resize(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad, unsigned flags,
                                const b200jpg_rect *rects, const b200jpg_size *sizes, int resample, b200jpg_batch **out) {
    return b200jpg_batch_create_draft(ctx, frames, lens, n, tolerate_bad, flags, nullptr, rects, sizes, resample, out);
}

int b200jpg_batch_create_draft(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad, unsigned flags,
                               const b200jpg_size *drafts, const b200jpg_rect *rects, const b200jpg_size *sizes, int resample, b200jpg_batch **out) {
    return b200jpg_batch_create_resample(ctx, frames, lens, n, tolerate_bad, flags, drafts, rects, sizes, nullptr, nullptr, resample, 0.0, out);
}

int b200jpg_batch_create_resample(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad, unsigned flags,
                                  const b200jpg_size *drafts, const b200jpg_rect *rects, const b200jpg_size *sizes, const b200jpg_box *boxes,
                                  const b200jpg_rect *windows, int resample, double reducing_gap, b200jpg_batch **out) {
    return b200jpg_batch_create_flip(ctx, frames, lens, n, tolerate_bad, flags, drafts, rects, sizes, boxes, windows, resample, reducing_gap,
                                     nullptr, out);
}

int b200jpg_batch_create_flip(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, int tolerate_bad, unsigned flags,
                              const b200jpg_size *drafts, const b200jpg_rect *rects, const b200jpg_size *sizes, const b200jpg_box *boxes,
                              const b200jpg_rect *windows, int resample, double reducing_gap, const uint8_t *flips, b200jpg_batch **out) {
    if (!ctx) return B200JPG_ERR_INVALID_PARAMETER;
    try {  // no exception crosses the C ABI
        return batch_create_impl(ctx, frames, lens, n, tolerate_bad, flags, drafts, rects, sizes, boxes, windows, resample, reducing_gap, flips,
                                 out);
    } catch (const std::bad_alloc &) {
        if (out) *out = nullptr;
        return ctx->fail(B200JPG_ERR_OUT_OF_MEMORY, "out of host memory while preparing the batch");
    } catch (...) {
        if (out) *out = nullptr;
        return ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "unexpected failure while preparing the batch");
    }
}

int b200jpg_batch_frame_info(const b200jpg_batch *b, int i, b200jpg_frame_info *info) {
    if (!b || i < 0 || i >= b->n_user || !info) return B200JPG_ERR_INVALID_PARAMETER;
    *info = b->frames[i].info;
    return b->parse_status[i];
}

int b200jpg_batch_output_extent(const b200jpg_batch *b, int i, int c, uint32_t *width, uint32_t *height) {
    if (!b || i < 0 || i >= b->n_user || !width || !height) return B200JPG_ERR_INVALID_PARAMETER;
    if (b->parse_status[i] != 0) return b->parse_status[i];
    const b200jpg_frame_info &fi = b->frames[i].info;
    if (c < 0 || c >= (int)b->plan[i].out_ncomp) return B200JPG_ERR_INVALID_PARAMETER;
    const Extent e = out_extent(fi, c, b->flags, b->plan[i]);
    *width = (uint32_t)e.w;
    *height = (uint32_t)e.h;
    return B200JPG_OK;
}

int b200jpg_batch_output_components(const b200jpg_batch *b, int i) {
    if (!b || i < 0 || i >= b->n_user) return B200JPG_ERR_INVALID_PARAMETER;
    if (b->parse_status[i] != 0) return b->parse_status[i];
    return (int)b->plan[i].out_ncomp;
}

int b200jpg_batch_frame_orientation(const b200jpg_batch *b, int i) {
    if (!b || i < 0 || i >= b->n_user) return B200JPG_ERR_INVALID_PARAMETER;
    return b->parse_status[i] != 0 ? b->parse_status[i] : b->frames[i].orientation;
}

uint64_t b200jpg_batch_out_offset(const b200jpg_batch *b, int i) { return (b && i >= 0 && i < b->n_user) ? b->out_off[i] : 0; }
uint64_t b200jpg_batch_out_bytes(const b200jpg_batch *b, int i) {
    if (!b) return 0;
    if (i < 0) return b->out_total;
    return i < b->n_user ? b->out_bytes[i] : 0;
}
uint64_t b200jpg_batch_ecs_bytes(const b200jpg_batch *b) { return b ? b->ecs_bytes : 0; }
uint64_t b200jpg_batch_stored_blocks(const b200jpg_batch *b) { return b ? b->stored_blocks : 0; }
uint64_t b200jpg_batch_h2d_bytes(const b200jpg_batch *b) { return b ? b->input_bytes : 0; }

uint64_t b200jpg_batch_export_tables(const b200jpg_batch *b, uint8_t *dst, uint64_t capacity) {
    if (!b || b->table_sets.size() != 1) return 0;
    const auto &blob = b->table_sets[0].blob;
    if (dst && capacity >= blob.size()) memcpy(dst, blob.data(), blob.size());
    return blob.size();
}

int b200jpg_batch_import_tables(b200jpg_batch *b, const uint8_t *src, uint64_t size) {
    if (!b || !src) return B200JPG_ERR_INVALID_PARAMETER;
    if (b->table_sets.size() != 1) return b->ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "table import needs a batch with exactly one table set");
    auto &blob = b->table_sets[0].blob;
    uint32_t hdr[4];
    if (size < 16) return b->ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "table blob too small");
    memcpy(hdr, src, 16);
    if (hdr[0] != kTableMagic || hdr[1] != size || size != blob.size())
        return b->ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "table blob does not match this batch (different table geometry)");
    memcpy(blob.data(), src, size);
    memcpy(b->h_input + b->dev_tables[0], src, size);
    b->uploaded = false;
    return B200JPG_OK;
}

// the restart index of device-indexed scans (restart_index_kernel): depends only on the uploaded bytes
static int run_restart_index(b200jpg_batch *b, void *stream) {
    uint32_t *index_status = b->d_status + 4 * (size_t)b->n + 1;
    cudaError_t e = cudaMemsetAsync(index_status, 0, sizeof(uint32_t) * (size_t)b->n, (cudaStream_t)stream);
    if (e != cudaSuccess) return b->ctx->fail_cuda(e, "index status reset");
    if (!b->index_scans.empty()) {
        int rc = launch_restart_index(reinterpret_cast<const IndexScan *>(b->d_input + b->dev_index_scans), (uint32_t)b->index_scans.size(),
                                      b->d_input, index_status, stream);
        if (rc != 0) return b->ctx->fail_cuda((cudaError_t)rc, "restart index kernel launch");
    }
    cudaEventRecord(b->ev_last, (cudaStream_t)stream);
    return B200JPG_OK;
}

int b200jpg_batch_upload(b200jpg_batch *b, void *stream) {
    NvtxRange nvtx("b200jpg upload: H2D + restart index");
    if (!b) return B200JPG_ERR_INVALID_PARAMETER;
    cudaSetDevice(b->ctx->device);
    cudaError_t e = cudaMemcpyAsync(b->d_input, b->h_input, b->input_bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream);
    if (e != cudaSuccess) return b->ctx->fail_cuda(e, "upload");
    int rc = run_restart_index(b, stream);  // built once per upload, right behind the copy
    if (rc) return rc;
    b->uploaded = true;
    return B200JPG_OK;
}

int b200jpg_batch_reindex(b200jpg_batch *b, void *stream) {
    if (!b) return B200JPG_ERR_INVALID_PARAMETER;
    if (!b->uploaded) return b->ctx->fail(B200JPG_ERR_OBJECT_DOESNT_EXIST, "batch has not been uploaded");
    cudaSetDevice(b->ctx->device);
    return run_restart_index(b, stream);
}

static int run_entropy(b200jpg_batch *b, void *stream) {
    NvtxRange nvtx("b200jpg entropy: unstuff + Huffman decode");
    // the status words start from what the restart index found at upload (out-of-sequence restart markers)
    cudaError_t e = cudaMemcpyAsync(b->d_status, b->d_status + 4 * (size_t)b->n + 1, sizeof(uint32_t) * (size_t)b->n, cudaMemcpyDeviceToDevice,
                                    (cudaStream_t)stream);
    if (e != cudaSuccess) return b->ctx->fail_cuda(e, "status reset");
    if (!b->prog_frames.empty() || b->clear_coef) {  // progressive scans accumulate into the coefficient store: it starts from zero
        e = cudaMemsetAsync(b->d_coef, 0, b->coef_elems * sizeof(int16_t), (cudaStream_t)stream);
        if (e != cudaSuccess) return b->ctx->fail_cuda(e, "coefficient store reset");
    }
    for (size_t ci = 0; ci < b->classes.size(); ci++) {  // the overrun lists start empty
        e = cudaMemsetAsync(b->d_overrun + b->classes[ci].interval_base + ci, 0, sizeof(uint32_t), (cudaStream_t)stream);
        if (e != cudaSuccess) return b->ctx->fail_cuda(e, "overrun list reset");
    }
    for (int pass = 0; pass < 2; pass++) {  // a0 for every class, then a1 for every class
        if (pass == 1 && b->timing && b->ev[3]) cudaEventRecord(b->ev[3], (cudaStream_t)stream);
        for (size_t ci = 0; ci < b->classes.size(); ci++) {
            auto &cl = b->classes[ci];
            EntropyLaunch l{};
            l.overrun_list = b->d_overrun + cl.interval_base + ci;
            l.p = cl.p;
            l.bytes = b->d_input;
            l.interval_off = reinterpret_cast<const uint64_t *>(b->d_input + cl.dev_intervals);
            l.interval_end = reinterpret_cast<const uint64_t *>(b->d_input + cl.dev_interval_end);
            l.clean_off = reinterpret_cast<const uint64_t *>(b->d_input + cl.dev_clean_off);
            l.clean = b->d_clean;
            l.interval_len = b->d_interval_len + cl.interval_base;
            l.scans = reinterpret_cast<const ClassScan *>(b->d_input + cl.dev_scans);
            l.tables = b->d_input + b->dev_tables[cl.table_set];
            l.coef = b->d_coef;
            l.frame_status = b->d_status;
            if (pass == 1 && cl.fused) continue;  // decoded by the component-fused launches below
            if (cl.p.indexed) {  // slices of the spec arrays: [segments | exits | entries | counts | dc sums], each over all work items
                const uint64_t n = align_up(b->n_spec, 4), o = cl.spec_base;  // (every slice starts 16-byte aligned)
                uint8_t *q = b->d_spec;
                l.spec_segments = reinterpret_cast<SpecSegment *>(q) + o;
                q += n * sizeof(SpecSegment);
                l.spec_exits = reinterpret_cast<unsigned long long *>(q) + o;
                q += n * 8;
                l.spec_entries = reinterpret_cast<unsigned long long *>(q) + o;
                q += n * 8;
                l.spec_counts = reinterpret_cast<uint32_t *>(q) + o;
                q += n * 4;
                l.spec_dc_sums = reinterpret_cast<int32_t *>(q) + 4 * o;
                q += n * 16;
                l.spec_logs = reinterpret_cast<SpecLog *>(q) + o;
                if (pass == 1) {
                    int rs = launch_spec_sync(l, stream);
                    if (rs != 0) return b->ctx->fail_cuda((cudaError_t)rs, "synchronisation kernel launch");
                    b->last_launches++;
                }
            }
            int rc = pass == 0 ? launch_unstuff(l, stream) : (cl.p.progressive ? launch_progressive_scan(l, stream) : launch_entropy(l, stream));
            if (rc != 0) return b->ctx->fail_cuda((cudaError_t)rc, pass == 0 ? "unstuff kernel launch" : "entropy kernel launch");
            b->last_launches++;
            if (pass == 1 && !cl.p.progressive && !cl.p.indexed) {
                rc = launch_overrun_verdict(l, stream);
                if (rc != 0) return b->ctx->fail_cuda((cudaError_t)rc, "overrun verdict kernel launch");
                b->last_launches++;
            }
        }
    }
    // ---- progressive frames decoded component by component: the DC scans into the side plane, then every component's AC scans
    for (size_t gi = 0; gi < b->pf_groups.size(); gi++) {
        const PfGroupHost &grp = b->pf_groups[gi];
        auto fill_scan = [&](PfScan &ps, const ScanClass &cl) {
            ps.tables = b->d_input + b->dev_tables[cl.table_set];
            ps.clean_off = reinterpret_cast<const uint64_t *>(b->d_input + cl.dev_clean_off);
            ps.interval_len = b->d_interval_len + cl.interval_base;
            ps.ss = cl.p.ss, ps.se = cl.p.se, ps.ah = cl.p.ah, ps.al = cl.p.al;
            for (int k = 0; k < 4; k++) ps.dc_slot[k] = cl.p.dc_slot[k];
            ps.ac_slot = cl.p.ac_slot[0];
            ps.q_slot = cl.p.q_slot[0];
            ps.lut_words = cl.p.lut_words;
        };
        auto fill_geometry = [&](PfLaunch &L, const ScanClass &cl) {
            L.ns = cl.p.ns;
            for (int k = 0; k < 4; k++) L.mw[k] = cl.p.mw[k], L.mh[k] = cl.p.mh[k], L.bw[k] = cl.p.bw[k];
            L.mcu_cols = cl.p.mcu_cols, L.total_mcus = cl.p.total_mcus, L.dri = cl.p.dri, L.intervals = cl.p.intervals_per_scan;
            L.n_frames = (uint32_t)cl.scans.size();
            L.frames = reinterpret_cast<const ClassScan *>(b->d_input + cl.dev_scans);
            L.clean = b->d_clean, L.coef = b->d_coef, L.dcplane = b->d_dcplane, L.frame_status = b->d_status;
        };
        {
            PfLaunch L{};
            L.n_scans = (int)grp.dc.size();
            for (size_t s = 0; s < grp.dc.size(); s++) fill_scan(L.scan[s], b->classes[(size_t)grp.dc[s]]);
            const ScanClass &dc0 = b->classes[(size_t)grp.dc[0]];
            fill_geometry(L, dc0);
            // scan component k of the DC scans is frame component comp[k] of the SOS: its quantiser and the block grid that
            // component's own AC scans cover (a component without AC scans is completed by the DC kernel alone)
            const ParsedFrame &pf0 = b->frames[dc0.scans[0].frame];
            for (int k = 0; k < L.ns; k++) {
                const int ci = pf0.scans[(size_t)dc0.p.ordinal].comp[k];
                L.ac_cols[k] = L.ac_rows[k] = 0;
                L.dc_quant[k] = b->pf_dc_quant[4 * gi + (size_t)ci];
                if (!grp.ac[ci].empty()) {
                    const ScanClassParams &ap = b->classes[(size_t)grp.ac[ci][0]].p;
                    L.ac_cols[k] = ap.mcu_cols;
                    L.ac_rows[k] = ap.total_mcus / ap.mcu_cols;
                }
            }
            int rc = launch_pf_dc(L, stream);
            if (rc != 0) return b->ctx->fail_cuda((cudaError_t)rc, "progressive DC kernel launch");
            b->last_launches++;
        }
        for (int c = 0; c < 4; c++) {
            if (grp.ac[c].empty()) continue;
            PfLaunch L{};
            L.n_scans = (int)grp.ac[c].size();
            for (size_t s = 0; s < grp.ac[c].size(); s++) {
                fill_scan(L.scan[s], b->classes[(size_t)grp.ac[c][s]]);
                // scans that decode with the same Huffman tables (the usual case: one AC table per component, or the
                // standard tables) share one copy in shared memory; the quantiser pairs differ with the point transform
                L.scan[s].lut_share = (int)s;
                const std::vector<uint8_t> &mine = b->table_sets[(size_t)b->classes[(size_t)grp.ac[c][s]].table_set].blob;
                for (size_t t = 0; t < s; t++) {
                    const std::vector<uint8_t> &other = b->table_sets[(size_t)b->classes[(size_t)grp.ac[c][t]].table_set].blob;
                    if (L.scan[t].lut_share == (int)t && L.scan[t].lut_words == L.scan[s].lut_words && L.scan[t].ac_slot == L.scan[s].ac_slot &&
                        mine.size() == other.size() && memcmp(mine.data() + 16, other.data() + 16, 16) == 0 &&
                        memcmp(mine.data() + kTableHeaderBytes, other.data() + kTableHeaderBytes, (size_t)L.scan[s].lut_words * 4) == 0) {
                        L.scan[s].lut_share = (int)t;
                        break;
                    }
                }
            }
            fill_geometry(L, b->classes[(size_t)grp.ac[c][0]]);
            L.dc_quant[0] = b->pf_dc_quant[4 * gi + (size_t)c];
            int rc = launch_pf_ac(L, stream);
            if (rc != 0) return b->ctx->fail_cuda((cudaError_t)rc, "progressive AC kernel launch");
            b->last_launches++;
        }
    }
    if (!b->prog_frames.empty()) {  // quantised levels -> the dequantised coefficients stage b expects
        int rc = launch_progressive_dequant(reinterpret_cast<const ProgFrame *>(b->d_input + b->dev_prog_frames), (uint32_t)b->prog_frames.size(),
                                            b->prog_max_blocks, b->d_coef, b->d_status, stream);
        if (rc != 0) return b->ctx->fail_cuda((cudaError_t)rc, "progressive dequantisation kernel launch");
        b->last_launches++;
    }
    cudaEventRecord(b->ev_last, (cudaStream_t)stream);
    return B200JPG_OK;
}

// The descriptor table [b->n_planes()] that fill(table) writes (on zeros: residual codestreams and failed frames have no destination) to
// b->d_planes on `stream`, staged in the next slot of the pinned ring (b200jpg_batch::kPlaneSlots); with `table` (the 4 KB of
// b200jpg_batch_decode_into_table) also the sample tables, at b->table_offset() of the slot, in the same copy
static int stage_planes(b200jpg_batch *b, void *stream, const std::function<void(b200jpg_plane *)> &fill, const float *table = nullptr) {
    const size_t bytes = sizeof(b200jpg_plane) * b->n_planes();
    const uint64_t slot_bytes = b->slot_bytes();
    cudaError_t ce = cudaSuccess;
    constexpr int kSlots = b200jpg_batch::kPlaneSlots;
    if (!b->d_planes) {  // everything is allocated before any of it is kept: a failure leaves the batch as it was
        b200jpg_plane *h = (b200jpg_plane *)b->ctx->get(0, slot_bytes * kSlots, &ce), *d = nullptr;
        cudaEvent_t ev[kSlots] = {};
        if (ce == cudaSuccess) d = (b200jpg_plane *)b->ctx->get(1, slot_bytes, &ce);
        for (int k = 0; k < kSlots && ce == cudaSuccess; k++) ce = cudaEventCreateWithFlags(&ev[k], cudaEventDisableTiming);
        if (ce != cudaSuccess) {
            const std::string why = cudaGetErrorString(ce);
            b->ctx->put(0, h, slot_bytes * kSlots);
            b->ctx->put(1, d, slot_bytes);
            for (auto &e : ev)
                if (e) cudaEventDestroy(e);
            return b->ctx->fail(B200JPG_ERR_OUT_OF_MEMORY, "descriptor table allocation failed: " + why);
        }
        b->h_planes = h, b->d_planes = d;
        for (int k = 0; k < kSlots; k++) b->ev_planes[k] = ev[k];
    }
    const int slot = b->plane_slot;
    ce = cudaEventSynchronize(b->ev_planes[slot]);  // the copy kSlots calls ago has read this slot (at once when never recorded)
    if (ce != cudaSuccess) return b->ctx->fail_cuda(ce, "descriptor table");
    uint8_t *base = reinterpret_cast<uint8_t *>(b->h_planes) + slot_bytes * slot;
    b200jpg_plane *stage = reinterpret_cast<b200jpg_plane *>(base);
    memset(stage, 0, bytes);
    fill(stage);
    if (table) memcpy(base + b->table_offset(), table, b200jpg_batch::kTableBytes);
    ce = cudaMemcpyAsync(b->d_planes, stage, table ? slot_bytes : bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream);
    if (ce == cudaSuccess) ce = cudaEventRecord(b->ev_planes[slot], (cudaStream_t)stream);
    b->plane_slot = (slot + 1) % kSlots;
    if (ce != cudaSuccess) return b->ctx->fail_cuda(ce, "descriptor table upload");
    return B200JPG_OK;
}

// Frame i's destinations, described in its output coordinates, rewritten into the decoded coordinates the kernels walk, in place:
// translated by its crop rectangle into the uncropped output (translate_plane), then oriented (orient_plane); planar[i] cleared
// unless every component then has bytes_per_pixel == size. Returns false when a pixel stride does not fit (only a caller's
// descriptor can do that). nc: the descriptors the reconstruction stores through (the plan's output components, or C's in the
// scratch).
static bool rewrite_frame(const b200jpg_batch *b, int i, b200jpg_plane *pl, uint64_t size, std::vector<char> &planar, uint32_t nc) {
    const FramePlan &p = b->plan[i];
    for (uint32_t c = 0; c < nc; c++) {
        const Extent d = decoded_extent(b->frames[i].info, c, b->flags, p.k);
        if (p.cropped) translate_plane(pl[c], p.crop);
        if (!orient_plane(pl[c], p.orientation, d.w, d.h)) return false;
        if ((uint64_t)pl[c].bytes_per_pixel != size) planar[(size_t)i] = 0;
    }
    return true;
}

// Live frame i's destinations q, described in its output coordinates (a caller's, or its packed slot's), made the ones its
// reconstruction stores through, in place: a resized frame's C in the scratch, an interleaved uint8 bitmap (its own destinations go
// to the resample pass: stage_frame_planes), rewritten like a cropped frame's; another described frame's rewritten (rewrite_frame),
// planar[i] decided on those; an undescribed frame's as they are. size: the bytes of a sample in q. Returns false as rewrite_frame.
static bool place_frame(const b200jpg_batch *b, int i, b200jpg_plane *q, uint64_t size, std::vector<char> &planar) {
    const FramePlan &p = b->plan[i];
    if (p.resized) {
        const ResampleFrame &f = b->rs_frames[(size_t)p.rs];
        for (uint32_t c = 0; c < f.ncomp; c++) {
            q[c].data = b->d_scratch + f.c_src + c;
            q[c].bytes_per_pixel = (int32_t)f.ncomp;
            q[c].bytes_per_row = f.c_pitch;
        }
        return rewrite_frame(b, i, q, 1, planar, f.ncomp);  // (a scratch row always fits the pixel stride)
    }
    if (!p.described) return true;
    planar[(size_t)i] = 1;
    return rewrite_frame(b, i, q, size, planar, p.out_ncomp);
}

// The descriptor table of a decode (staged: stage_planes): every live frame's placed destinations q (place_frame), and the
// destinations of resized frame r, as given in `planes`, at 4 * (n + r) for the resample pass ([4 * n_user] each), mirrored over
// the window's tw x th for a flipped frame (flip_plane); the sample tables behind them (stage_planes)
static int stage_frame_planes(b200jpg_batch *b, const b200jpg_plane *q, const b200jpg_plane *planes, void *stream, const float *table = nullptr) {
    return stage_planes(b, stream, [&](b200jpg_plane *table) {
        for (int i = 0; i < b->n_user; i++) {
            const FramePlan &p = b->plan[i];
            if (b->parse_status[i] != 0) continue;
            memcpy(table + 4 * (size_t)i, q + 4 * (size_t)i, sizeof(b200jpg_plane) * p.out_ncomp);
            if (!p.resized) continue;
            b200jpg_plane *rs = table + 4 * ((size_t)b->n + p.rs);
            memcpy(rs, planes + 4 * (size_t)i, sizeof(b200jpg_plane) * p.out_ncomp);
            const ResampleFrame &f = b->rs_frames[(size_t)p.rs];
            for (uint32_t c = 0; p.flip && c < p.out_ncomp; c++) flip_plane(rs[c], p.flip, f.tw, f.th);
        }
    }, table);
}

// b200jpg_batch_decode of a batch with described frames: each such frame's packed slot in out_dev, described as a caller of
// b200jpg_batch_decode_into would: an interleaved bitmap of its output extent (B200JPG_FLAG_NO_UPSAMPLE: plane after plane), placed
// and staged as that call's table is (never checked like it). planar[i] as for that table.
static int stage_slot_planes(b200jpg_batch *b, uint8_t *out_dev, void *stream, std::vector<char> &planar) {
    std::vector<b200jpg_plane> slots(4 * (size_t)b->n_user), q(slots.size());
    for (int i = 0; i < b->n_user; i++) {
        const FramePlan &p = b->plan[i];
        if (b->parse_status[i] != 0 || !p.described) continue;
        const b200jpg_frame_info &fi = b->frames[i].info;
        const int64_t size = fi.precision > 8 ? 2 : 1;
        const bool planes = (b->flags & B200JPG_FLAG_NO_UPSAMPLE) != 0;
        uint64_t before = 0;
        b200jpg_plane *pl = &slots[4 * (size_t)i];
        for (uint32_t c = 0; c < p.out_ncomp; c++) {
            const Extent e = out_extent(fi, (int)c, b->flags, p);
            pl[c].data = out_dev + b->out_off[i] + (planes ? before : (uint64_t)c) * size;
            pl[c].bytes_per_pixel = (int32_t)(planes ? size : p.out_ncomp * size);
            pl[c].bytes_per_row = (int64_t)e.w * pl[c].bytes_per_pixel;
            before += e.w * e.h;
        }
        std::copy_n(pl, 4, &q[4 * (size_t)i]);
        place_frame(b, i, &q[4 * (size_t)i], (uint64_t)size, planar);  // (a slot's row stride always fits the pixel stride)
    }
    return stage_frame_planes(b, q.data(), slots.data(), stream);
}

// planes_dev: b200jpg_batch_decode_into's descriptor table (device), planar[i]: every component of frame i has
// bytes_per_pixel == sample size (element size with `convert`, the float map of b200jpg_batch_decode_into_ex); table: with
// `convert`, the sample tables of b200jpg_batch_decode_into_table (device)
static int run_recon(b200jpg_batch *b, uint8_t *out_dev, void *stream, const b200jpg_plane *planes_dev = nullptr,
                     const std::vector<char> *planar = nullptr, const b200jpg_convert *convert = nullptr, const float *table = nullptr) {
    NvtxRange nvtx("b200jpg reconstruction: IDCT + upsampling + colour");
    // into the packed slots with described frames: those frames' slots as descriptors, built for this call's out_dev; the groups of
    // the other frames store into out_dev
    std::vector<char> slot_planar;
    if (!planes_dev && b->rewritten) {
        slot_planar.assign((size_t)b->n, 1);
        if (int rc = stage_slot_planes(b, out_dev, stream, slot_planar)) return rc;
        planes_dev = b->d_planes, planar = &slot_planar;
    }
    cudaError_t me = cudaMemsetAsync(b->d_status + b->n, 0, sizeof(uint32_t) * 2 * (size_t)b->n, (cudaStream_t)stream);
    if (me != cudaSuccess) return b->ctx->fail_cuda(me, "flag reset");
    for (auto &g : b->groups) {
        ReconLaunch l{};
        l.frames = reinterpret_cast<const FrameRecon *>(b->d_input + g.dev_frames);
        l.n_frames = (uint32_t)g.frames.size();
        l.max_bw0 = g.max_bw0;
        l.max_bh0 = g.max_bh0;
        l.max_bwc = g.max_bwc;
        l.max_bhc = g.max_bhc;
        l.ncomp = g.key.ncomp;
        l.subx = g.key.subx;
        l.suby = g.key.suby;
        l.path = g.key.path;
        l.mode = g.key.mode;
        l.downscale = (int)g.key.scale;
        l.planes_out = (b->flags & B200JPG_FLAG_NO_UPSAMPLE) != 0;
        l.coef = b->d_coef;
        l.samples16 = b->d_samples16;
        l.samples32 = b->d_samples;
        l.planes8 = b->d_planes8;
        l.wide_flags = b->d_status + b->n;
        l.narrow_flags = b->d_status + 2 * (size_t)b->n;
        l.narrow_list = b->d_status + 3 * (size_t)b->n;
        l.out = out_dev;
        l.planes = (out_dev && !g.key.described) ? nullptr : planes_dev;
        l.convert = convert;
        l.table = table;
        if (g.key.resized) l.convert = nullptr, l.table = nullptr;  // C leaves as uint8; the resample pass converts
        l.planar = l.planes != nullptr;
        if (l.planes)
            for (const FrameRecon &fr : g.frames) l.planar = l.planar && (*planar)[fr.status_idx];
        // oriented frames into anything but planar destinations: the staged store kinds, runs of eight samples along x or y; cropped
        // frames into any destination: the same kinds with the clip (the generic kernels: the strided kinds with the clip)
        l.runs = g.key.described && l.planes && (!l.planar || g.key.cropped);
        l.clip = g.key.cropped;
        int launches = 0;
        // grid.y carries the frame index: at most 65535 frames per launch. A generic group that is cut runs the IDCT of ALL its
        // frames first: a JPEG XT frame reads the planes of its residual frame, which may sit in another part
        const bool cut = l.path == ReconPath::Generic && l.n_frames > 65535u;
        for (int phase = cut ? 1 : 0; phase <= (cut ? 2 : 0); phase++) {
            for (uint32_t first = 0; first < l.n_frames; first += 65535u) {
                ReconLaunch part = l;
                part.frames = l.frames + first;
                part.n_frames = std::min<uint32_t>(65535u, l.n_frames - first);
                part.generic_phase = phase;
                int rc = launch_recon(part, stream, &launches);
                if (rc != 0) return b->ctx->fail_cuda((cudaError_t)rc, "reconstruction kernel launch");
                b->last_launches += launches;
            }
        }
    }
    // resized frames: C in the scratch -> the destinations (grid.y carries the frame: at most 65535 frames per launch)
    const uint32_t nr = (uint32_t)b->rs_frames.size();
    for (uint32_t first = 0; first < nr; first += 65535u) {
        ResampleLaunch rl{};
        rl.frames = reinterpret_cast<const ResampleFrame *>(b->d_input + b->dev_rs_frames) + first;
        rl.n_frames = std::min<uint32_t>(65535u, nr - first);
        rl.max_rows = b->rs_max_rows;
        rl.max_reduce_rows = b->rs_max_reduce_rows;
        rl.max_pixels = b->rs_max_pixels;
        rl.input = b->d_input;
        rl.scratch = b->d_scratch;
        rl.inter = b->d_inter;
        rl.planes = planes_dev;
        rl.convert = convert;
        rl.table = table;
        rl.n_plain = std::min(rl.n_frames, b->rs_plain > first ? b->rs_plain - first : 0u);
        rl.resample = b->resample;
        rl.cv_kinds = b->rs_cv_kinds;
        int launches = 0;
        int rc = launch_resample(rl, stream, &launches);
        if (rc != 0) return b->ctx->fail_cuda((cudaError_t)rc, "resample kernel launch");
        b->last_launches += launches;
    }
    cudaEventRecord(b->ev_last, (cudaStream_t)stream);
    return B200JPG_OK;
}

static int ensure_events(b200jpg_batch *b) {
    for (auto &e : b->ev)
        if (!e && cudaEventCreate(&e) != cudaSuccess) return b->ctx->fail(B200JPG_ERR_CUDA, "cudaEventCreate failed");
    return 0;
}

static int run_decode(b200jpg_batch *b, uint8_t *out_dev, void *stream, const b200jpg_plane *planes_dev = nullptr,
                      const std::vector<char> *planar = nullptr, const b200jpg_convert *convert = nullptr, const float *table = nullptr) {
    b->last_launches = 0;
    b->status_fetched = false;
    if (b->timing) {
        if (ensure_events(b)) return B200JPG_ERR_CUDA;
        cudaEventRecord(b->ev[0], (cudaStream_t)stream);
    }
    int rc = run_entropy(b, stream);
    if (rc) return rc;
    if (b->timing) cudaEventRecord(b->ev[1], (cudaStream_t)stream);
    rc = run_recon(b, out_dev, stream, planes_dev, planar, convert, table);
    if (rc) return rc;
    if (b->timing) cudaEventRecord(b->ev[2], (cudaStream_t)stream);
    return B200JPG_OK;
}

int b200jpg_batch_decode(b200jpg_batch *b, uint8_t *out_dev, void *stream) {
    if (!b || !out_dev) return B200JPG_ERR_INVALID_PARAMETER;
    if (!b->uploaded) return b->ctx->fail(B200JPG_ERR_OBJECT_DOESNT_EXIST, "batch has not been uploaded");
    cudaSetDevice(b->ctx->device);
    return run_decode(b, out_dev, stream);
}

static uint64_t magnitude(int64_t v) { return v < 0 ? 0 - (uint64_t)v : (uint64_t)v; }

int b200jpg_batch_decode_into(b200jpg_batch *b, const b200jpg_plane *planes, void *stream) {
    return b200jpg_batch_decode_into_ex(b, planes, nullptr, stream);
}

// the bytes of one float element of B200JPG_SAMPLE_* `type`; 0 for an unknown type
static uint64_t element_size(int32_t type) {
    return type == B200JPG_SAMPLE_F32 ? 4 : ((type == B200JPG_SAMPLE_F16 || type == B200JPG_SAMPLE_BF16) ? 2 : 0);
}

// b200jpg_batch_decode_into(_ex, _table) once the map is checked: every descriptor of every live frame is checked before anything
// is enqueued, then placed, staged (with the sample tables of `table`, host) and decoded into
static int decode_into_checked(b200jpg_batch *b, const b200jpg_plane *planes, const b200jpg_convert *convert, const float *table, void *stream) {
    const uint64_t element = convert ? element_size(convert->type) : 0;  // float destinations: the element size replaces the sample size
    std::vector<char> planar((size_t)b->n, 1);
    std::vector<b200jpg_plane> q(planes, planes + 4 * (size_t)b->n_user);  // placed once here (place_frame)
    for (int i = 0; i < b->n_user; i++) {
        if (b->parse_status[i] != 0) continue;
        const b200jpg_frame_info &fi = b->frames[i].info;
        const uint64_t size = convert ? element : (fi.precision > 8 ? 2 : 1);
        const FramePlan &plan = b->plan[i];
        for (int c = 0; c < (int)plan.out_ncomp; c++) {
            const b200jpg_plane &p = planes[4 * i + c];
            const auto [w, h] = out_extent(fi, c, b->flags, plan);  // the rules hold in (cropped, resized) output coordinates
            const uint64_t bpp = magnitude(p.bytes_per_pixel), bpr = magnitude(p.bytes_per_row);
            const std::string at = "frame " + std::to_string(i) + " component " + std::to_string(c) + ": ";
            if (!p.data) return b->ctx->fail(B200JPG_ERR_INVALID_PARAMETER, at + "no destination");
            if (bpp < size) return b->ctx->fail(B200JPG_ERR_INVALID_PARAMETER, at + "|bytes_per_pixel| is smaller than the sample size");
            if (h > 1 && bpr < w * bpp) return b->ctx->fail(B200JPG_ERR_INVALID_PARAMETER, at + "rows overlap: |bytes_per_row| < width * |bytes_per_pixel|");
            if (size > 1 && ((reinterpret_cast<uintptr_t>(p.data) | bpp | bpr) & (size - 1u)))
                return b->ctx->fail(B200JPG_ERR_INVALID_PARAMETER,
                                    at + (convert ? std::to_string(size) + "-byte elements need a " + std::to_string(size) + "-byte aligned address and strides"
                                                  : std::string("16-bit samples need a 2-byte aligned address and strides")));
            cudaPointerAttributes a{};
            const cudaError_t e = cudaPointerGetAttributes(&a, p.data);
            if (e != cudaSuccess) cudaGetLastError();
            if (e != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != b->ctx->device)
                return b->ctx->fail(B200JPG_ERR_INVALID_PARAMETER, at + "not device memory of the batch's device");
            if ((uint64_t)p.bytes_per_pixel != size) planar[(size_t)i] = 0;
        }
        if (!place_frame(b, i, &q[4 * (size_t)i], size, planar))
            return b->ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "frame " + std::to_string(i) + ": |bytes_per_row| does not fit the pixel stride of the transposed frame");
    }
    if (int rc = stage_frame_planes(b, q.data(), planes, stream, table)) return rc;
    const float *table_dev = table ? reinterpret_cast<const float *>(reinterpret_cast<uint8_t *>(b->d_planes) + b->table_offset()) : nullptr;
    return run_decode(b, nullptr, stream, b->d_planes, &planar, convert, table_dev);
}

int b200jpg_batch_decode_into_ex(b200jpg_batch *b, const b200jpg_plane *planes, const b200jpg_convert *convert, void *stream) {
    if (!b || !planes) return B200JPG_ERR_INVALID_PARAMETER;
    if (!b->uploaded) return b->ctx->fail(B200JPG_ERR_OBJECT_DOESNT_EXIST, "batch has not been uploaded");
    cudaSetDevice(b->ctx->device);
    if (convert) {
        if (!element_size(convert->type)) return b->ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "unknown sample type " + std::to_string(convert->type));
        int ncomp = 0;  // the components some live frame is written with
        for (int i = 0; i < b->n_user; i++)
            if (b->parse_status[i] == 0) ncomp = std::max(ncomp, (int)b->plan[i].out_ncomp);
        for (int c = 0; c < ncomp; c++)
            if (!std::isfinite(convert->scale[c]) || !std::isfinite(convert->bias[c]))
                return b->ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "component " + std::to_string(c) + ": scale and bias must be finite");
    }
    return decode_into_checked(b, planes, convert, nullptr, stream);
}

int b200jpg_batch_decode_into_table(b200jpg_batch *b, const b200jpg_plane *planes, const b200jpg_convert_table *table, void *stream) {
    if (!b || !planes) return B200JPG_ERR_INVALID_PARAMETER;
    if (!b->uploaded) return b->ctx->fail(B200JPG_ERR_OBJECT_DOESNT_EXIST, "batch has not been uploaded");
    cudaSetDevice(b->ctx->device);
    if (!table) return b->ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "no sample table");
    if (!element_size(table->type)) return b->ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "unknown sample type " + std::to_string(table->type));
    for (int i = 0; i < b->n_user; i++)
        if (b->parse_status[i] == 0 && b->frames[i].info.precision > 8)
            return b->ctx->fail(B200JPG_ERR_NOT_IMPLEMENTED, "frame " + std::to_string(i) + ": 12-bit samples have no 256-entry sample table");
    b200jpg_convert convert{};  // the element type; the tables replace the map
    convert.type = table->type;
    return decode_into_checked(b, planes, &convert, &table->table[0][0], stream);
}

int b200jpg_batch_decode_entropy(b200jpg_batch *b, void *stream) {
    if (!b) return B200JPG_ERR_INVALID_PARAMETER;
    if (!b->uploaded) return b->ctx->fail(B200JPG_ERR_OBJECT_DOESNT_EXIST, "batch has not been uploaded");
    cudaSetDevice(b->ctx->device);
    b->last_launches = 0;
    b->status_fetched = false;
    return run_entropy(b, stream);
}

int b200jpg_batch_reconstruct(b200jpg_batch *b, uint8_t *out_dev, void *stream) {
    if (!b || !out_dev) return B200JPG_ERR_INVALID_PARAMETER;
    if (!b->uploaded) return b->ctx->fail(B200JPG_ERR_OBJECT_DOESNT_EXIST, "batch has not been uploaded");
    cudaSetDevice(b->ctx->device);
    b->last_launches = 0;
    return run_recon(b, out_dev, stream);
}

int b200jpg_batch_frame_status(b200jpg_batch *b, int i) {
    if (!b || i < 0 || i >= b->n_user) return B200JPG_ERR_INVALID_PARAMETER;
    if (b->parse_status[i] != 0) return b->parse_status[i];
    if (!b->status_fetched) {
        cudaSetDevice(b->ctx->device);
        cudaError_t e = cudaMemcpy(b->h_status.data(), b->d_status, sizeof(uint32_t) * (size_t)b->n, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) return b->ctx->fail_cuda(e, "status download");
        b->status_fetched = true;
    }
    if (b->h_status[i] == 0 && b->xt_child[i] >= 0) return -(int)b->h_status[b->xt_child[i]];  // JPEG XT: the residual codestream's errors are the frame's
    return -(int)b->h_status[i];
}

int b200jpg_batch_read_coefficients(b200jpg_batch *b, int i, int c, int16_t *dst, uint64_t capacity) {
    if (!b || i < 0 || i >= b->n || !dst) return B200JPG_ERR_INVALID_PARAMETER;
    if (b->parse_status[i] != 0) return b->parse_status[i];
    const b200jpg_frame_info &fi = b->frames[i].info;
    if (c < 0 || c >= fi.ncomp) return B200JPG_ERR_INVALID_PARAMETER;
    uint64_t elems = (uint64_t)fi.blocks_w[c] * fi.blocks_h[c] * 64;
    if (capacity < elems) return B200JPG_ERR_INVALID_PARAMETER;
    cudaSetDevice(b->ctx->device);
    cudaError_t e = cudaMemcpy(dst, b->d_coef + b->coef_base[i][c], elems * sizeof(int16_t), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return b->ctx->fail_cuda(e, "coefficient download");
    return B200JPG_OK;
}

int b200jpg_batch_last_launch_count(const b200jpg_batch *b) { return b ? b->last_launches : 0; }

void b200jpg_batch_enable_timing(b200jpg_batch *b, int on) {
    if (b) b->timing = on != 0;
}

float b200jpg_batch_last_unstuff_ms(b200jpg_batch *b) {
    float a = 0;
    if (!b || !b->ev[0] || !b->ev[3]) return -1.f;
    if (cudaEventElapsedTime(&a, b->ev[0], b->ev[3]) != cudaSuccess) return -1.f;
    return a;
}

int b200jpg_batch_last_timing(b200jpg_batch *b, float *entropy_ms, float *reconstruct_ms) {
    if (!b || !b->ev[0]) return B200JPG_ERR_INVALID_PARAMETER;
    float a = 0, c = 0;
    if (cudaEventElapsedTime(&a, b->ev[0], b->ev[1]) != cudaSuccess) return B200JPG_ERR_CUDA;
    if (cudaEventElapsedTime(&c, b->ev[1], b->ev[2]) != cudaSuccess) return B200JPG_ERR_CUDA;
    if (entropy_ms) *entropy_ms = a;
    if (reconstruct_ms) *reconstruct_ms = c;
    return B200JPG_OK;
}

// Scan 0 of a restart-less codestream as the host replay of spec_sync_kernel takes it (tests only)
struct ReplayScan {
    TableSet ts;
    SpecScan ss{};
    std::vector<uint32_t> words;
    uint32_t len_bytes = 0, total_mcus = 0;
    int ns = 0;
};

static int replay_scan0(const uint8_t *data, size_t len, ReplayScan &rs) {
    ParsedFrame pf;
    std::string err;
    int rc = parse_codestream(data, len, pf, err);
    if (rc) return rc;
    const ScanInfo &sc = pf.scans[0];
    if (sc.progressive || sc.interval_off.size() != 1) return B200JPG_ERR_INVALID_PARAMETER;
    TableSet &ts = rs.ts;
    rc = build_table_set(sc, ts, err);
    if (rc) return rc;
    // unstuff (io/bitstream.cpp:56-118) into big-endian words
    std::vector<uint8_t> bytes;
    for (size_t i = sc.ecs_off; i < sc.ecs_end; i++) {
        if (data[i] == 0xff) {
            if (i + 1 < sc.ecs_end && data[i + 1] == 0x00) {
                bytes.push_back(0xff);
                i++;
                continue;
            }
            break;  // a marker
        }
        bytes.push_back(data[i]);
    }
    rs.len_bytes = (uint32_t)bytes.size();
    bytes.resize((bytes.size() + 3) / 4 * 4 + 64, 0);
    std::vector<uint32_t> &words = rs.words;
    words.resize(bytes.size() / 4);
    for (size_t i = 0; i < words.size(); i++)
        words[i] = ((uint32_t)bytes[4 * i] << 24) | ((uint32_t)bytes[4 * i + 1] << 16) | ((uint32_t)bytes[4 * i + 2] << 8) | bytes[4 * i + 3];
    const uint16_t *lut_off = reinterpret_cast<const uint16_t *>(ts.blob.data() + 16);
    SpecScan &ss = rs.ss;
    ss.lut = reinterpret_cast<const uint32_t *>(ts.blob.data() + kTableHeaderBytes);
    const b200jpg_frame_info &fi = pf.info;
    for (int c = 0; c < sc.ns; c++) {
        ss.dc_tab[c] = lut_off[sc.td[c]];
        ss.ac_tab[c] = lut_off[4 + sc.ta[c]];
        const int nb = sc.ns > 1 ? fi.hs[sc.comp[c]] * fi.vs[sc.comp[c]] : 1;
        for (int k = 0; k < nb; k++) ss.comp_of_block[ss.blocks_per_mcu++] = (uint8_t)c;
    }
    ss.blk_period = ss.blocks_per_mcu;  // exact positions for the walks of the self-test; the replay finds its own period
    rs.total_mcus = sc.mcu_cols * sc.mcu_rows;
    rs.ns = sc.ns;
    return B200JPG_OK;
}

static int replay_rounds(const ReplayScan &rs, std::vector<SpecSegment> &segs) {
    extern unsigned long long g_spec_replay_bits, g_spec_replay_merges[kSpecMarks];
    g_spec_replay_bits = 0;
    for (auto &m : g_spec_replay_merges) m = 0;
    const int r = spec_sync_host_replay(rs.ss, rs.words.data(), rs.len_bytes, rs.total_mcus, segs);
    if (getenv("B200JPG_SPEC_STATS")) {
        fprintf(stderr, "restart-less replay: %u rounds, %.2f x the stream walked, merges at marks", (unsigned)r,
                (double)g_spec_replay_bits / (8.0 * rs.len_bytes + 1));
        for (int m = 0; m < kSpecMarks; m++) fprintf(stderr, " %llu", g_spec_replay_merges[m]);
        fprintf(stderr, "\n");
    }
    return r;
}

// Host replay of the synchronisation rounds of spec_sync_kernel on scan 0 of one codestream, checked against a plain
// front-to-back walk of the same stream (tests only: it validates the round logic, prefix sums and clipping that the device
// kernel shares through specsync.hpp; nothing in the decode path calls it).
int b200jpg_selftest_restartless(const uint8_t *data, size_t len, uint32_t *rounds, uint32_t *n_segments) {
    ReplayScan rs;
    const int rc = replay_scan0(data, len, rs);
    if (rc) return rc;
    const SpecScan &ss = rs.ss;
    const std::vector<uint32_t> &words = rs.words;
    const uint32_t len_bytes = rs.len_bytes, total_mcus = rs.total_mcus;
    std::vector<SpecSegment> segs;
    const int r = replay_rounds(rs, segs);
    if (rounds) *rounds = (uint32_t)r;
    if (n_segments) *n_segments = (uint32_t)segs.size();
    // the truth: one walk from the first bit, block by block
    const uint32_t total_blocks = total_mcus * ss.blocks_per_mcu, nwords = (len_bytes + 3) / 4;
    std::vector<uint32_t> start_bit(total_blocks + 1);
    std::vector<int32_t> pred_at((size_t)(total_blocks + 1) * 4, 0);
    SpecState st{0, 0};
    int32_t pred[4] = {0, 0, 0, 0};
    uint32_t walked = 0;
    for (; walked < total_blocks && st.bit < len_bytes * 8u; walked++) {
        start_bit[walked] = st.bit;
        for (int c = 0; c < 4; c++) pred_at[(size_t)walked * 4 + c] = pred[c];
        const SpecResult one = spec_decode(ss, words.data(), nwords, len_bytes * 8u, st, st.bit + 1);
        for (int c = 0; c < 4; c++) pred[c] += one.dc_sum[c];
        st = one.exit;
    }
    uint32_t covered = 0;
    for (const SpecSegment &g : segs) {
        if (g.n_blocks == 0) continue;
        if (g.first_block != covered) return -1;                       // the segments tile the blocks in order
        if (g.first_block < walked) {
            if (g.bit != start_bit[g.first_block]) return -2;          // and start where their first block starts
            for (int c = 0; c < rs.ns; c++)
                if (g.pred[c] != pred_at[(size_t)g.first_block * 4 + c]) return -3;  // with the predictors of that place
        }
        covered += g.n_blocks;
    }
    if (covered != total_blocks) return -4;
    return B200JPG_OK;
}

// The same replay's work items themselves (tests only), seven int32 each: start bit, first block, block count and the four
// DC predictors, for tests that hold them against what the encoder recorded rather than against another walk of the decoder.
int b200jpg_selftest_restartless_items(const uint8_t *data, size_t len, int32_t *items, uint32_t cap, uint32_t *n_items, uint32_t *rounds) {
    ReplayScan rs;
    const int rc = replay_scan0(data, len, rs);
    if (rc) return rc;
    std::vector<SpecSegment> segs;
    const int r = replay_rounds(rs, segs);
    if (rounds) *rounds = (uint32_t)r;
    if (n_items) *n_items = (uint32_t)segs.size();
    if (!items || segs.size() > cap) return B200JPG_ERR_INVALID_PARAMETER;
    for (size_t i = 0; i < segs.size(); i++) {
        int32_t *o = items + 7 * i;
        o[0] = (int32_t)segs[i].bit, o[1] = (int32_t)segs[i].first_block, o[2] = (int32_t)segs[i].n_blocks;
        for (int c = 0; c < 4; c++) o[3 + c] = segs[i].pred[c];
    }
    return B200JPG_OK;
}

int b200jpg_selftest_table_cache(const uint8_t *const *frames, const size_t *lens, int n) {
    if (!frames || !lens || n <= 0) return B200JPG_ERR_INVALID_PARAMETER;
    TableCache cache;
    int scans_checked = 0;
    for (int pass = 0; pass < 2; pass++)  // twice: the second time every scan comes out of the cache
        for (int i = 0; i < n; i++) {
            ParsedFrame pf;
            std::string err;
            if (parse_codestream(frames[i], lens[i], pf, err) != 0) continue;
            for (const ScanInfo &sc : pf.scans) {
                TableSet cached, fresh;
                std::string e1, e2;
                const int r1 = build_table_set_cached(sc, cached, e1, cache), r2 = build_table_set(sc, fresh, e2);
                if (r1 != r2) return -1;
                if (r1 == 0 && cached.blob != fresh.blob) return -2;
                scans_checked++;
            }
        }
    return scans_checked;
}

int b200jpg_decode_to_host(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, uint8_t *out_host,
                           uint64_t out_capacity) {
    return b200jpg_decode_to_host_ex(ctx, frames, lens, n, out_host, out_capacity, 0u);
}

// One-shot decode of n frames into a fresh device buffer: handed to the caller through out_dev / out_bytes, or without out_dev
// copied to out_host (its capacity checked first) and freed.
static int decode_once(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, unsigned flags, uint8_t *out_host,
                       uint64_t out_capacity, uint8_t **out_dev, uint64_t *out_bytes) {
    const bool to_host = out_dev == nullptr;
    b200jpg_batch *b = nullptr;
    int rc = b200jpg_batch_create_ex(ctx, frames, lens, n, 0, flags, &b);
    if (rc) return rc;
    uint8_t *d_out = nullptr;
    cudaStream_t s = nullptr;
    cudaError_t e = cudaSuccess;
    if (to_host && out_capacity < b->out_total) rc = ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "output buffer too small");
    if (!rc && cudaMalloc((void **)&d_out, b->out_total ? b->out_total : 1) != cudaSuccess)
        rc = ctx->fail(B200JPG_ERR_OUT_OF_MEMORY, "device allocation of the output failed");
    if (!rc && (e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)) != cudaSuccess) rc = ctx->fail_cuda(e, "cudaStreamCreate");
    if (!rc) rc = b200jpg_batch_upload(b, s);
    if (!rc) rc = b200jpg_batch_decode(b, d_out, s);
    if (!rc) {
        if (to_host) e = cudaMemcpyAsync(out_host, d_out, b->out_total, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) rc = ctx->fail_cuda(e, to_host ? "download" : "decode");
    }
    for (int i = 0; i < n && !rc; i++) {
        int st = b200jpg_batch_frame_status(b, i);
        if (st) rc = ctx->fail(st, "frame " + std::to_string(i) + ": invalid stream, found invalid huffman code in entropy coded segment");
    }
    if (!rc && !to_host) {
        if (out_bytes) *out_bytes = b->out_total;
        *out_dev = d_out;
        d_out = nullptr;
    }
    if (s) cudaStreamDestroy(s);
    if (d_out) cudaFree(d_out);
    b200jpg_batch_destroy(b);
    return rc;
}

int b200jpg_decode_to_host_ex(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, uint8_t *out_host,
                              uint64_t out_capacity, unsigned flags) {
    if (!ctx) return B200JPG_ERR_INVALID_PARAMETER;
    return decode_once(ctx, frames, lens, n, flags, out_host, out_capacity, nullptr, nullptr);
}

int b200jpg_decode_to_device_ex(b200jpg_ctx *ctx, const uint8_t *const *frames, const size_t *lens, int n, unsigned flags, uint8_t **out_dev,
                                uint64_t *out_bytes) {
    if (!ctx || !out_dev) return B200JPG_ERR_INVALID_PARAMETER;
    *out_dev = nullptr;
    return decode_once(ctx, frames, lens, n, flags, nullptr, 0, out_dev, out_bytes);
}

void b200jpg_device_free(b200jpg_ctx *ctx, uint8_t *p) {
    if (!p) return;
    if (ctx) cudaSetDevice(ctx->device);
    cudaFree(p);
}

int b200jpg_device_copy_rect(b200jpg_ctx *ctx, uint8_t *dst_dev, int64_t dst_pitch, const uint8_t *src_dev, int64_t src_pitch, uint64_t width_bytes,
                             uint64_t rows) {
    if (!ctx || !dst_dev || !src_dev || dst_pitch < 0 || src_pitch < 0) return B200JPG_ERR_INVALID_PARAMETER;
    if (width_bytes == 0 || rows == 0) return B200JPG_OK;
    cudaSetDevice(ctx->device);
    cudaError_t e = cudaMemcpy2D(dst_dev, (size_t)dst_pitch, src_dev, (size_t)src_pitch, (size_t)width_bytes, (size_t)rows, cudaMemcpyDeviceToDevice);
    if (e != cudaSuccess) return ctx->fail_cuda(e, "device rectangle copy");
    return B200JPG_OK;
}

}  // extern "C"

namespace b200jpg {
int device_bitmap_copy(b200jpg_ctx *ctx, const BitmapRequest &r, const uint8_t *src) {
    if (!ctx || !src) return B200JPG_ERR_INVALID_PARAMETER;
    cudaSetDevice(ctx->device);
    for (int k = 0; k < r.ncomp; k++) {
        if (!r.comp[k].dst) continue;
        cudaPointerAttributes a{};
        const cudaError_t e = cudaPointerGetAttributes(&a, r.comp[k].dst);
        if (e != cudaSuccess) cudaGetLastError();
        if (e != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != ctx->device)
            return ctx->fail(B200JPG_ERR_INVALID_PARAMETER, "device bitmaps: component " + std::to_string(k) + " is not device memory of the decoding device");
    }
    int rc = launch_bitmap_copy(r, src, nullptr);
    cudaError_t e = rc ? (cudaError_t)rc : cudaStreamSynchronize(nullptr);
    if (e != cudaSuccess) return ctx->fail_cuda(e, "device bitmap copy");
    return B200JPG_OK;
}
}  // namespace b200jpg
