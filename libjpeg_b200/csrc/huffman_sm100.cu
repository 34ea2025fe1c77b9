// huffman_sm100.cu -- stage (a): sequential-scan Huffman decode + dequantisation on sm_90a.
//
// Replaces the reference's entropy path for SOF0/SOF1 Huffman scans:
//   SequentialScan::ParseMCU / DecodeBlock / Restart   codestream/sequentialscan.cpp:381-428, 678-773, 266-274
//   EntropyParser::BeginReadMCU                        codestream/entropyparser.hpp:147-160
//   HuffmanDecoder::Get (two-level 8+8 bit lookup)     coding/huffmandecoder.hpp:103-124
//   BitStream<false>::Fill / Get / PeekWord / SkipBits io/bitstream.cpp:56-118, io/bitstream.hpp:168-208
//   dequantisation multiplier                          dct/idct.cpp:98-108 (the << 4 is left to stage b)
//
// The restart interval is the unit of work: each one restarts the bit reader byte-aligned and resets the DC
// predictors (sequentialscan.cpp:266-274), so intervals are independent.  Two kernels:
//
// a0  unstuff_kernel -- ONE WARP PER RESTART INTERVAL.  Streams the interval's entropy coded bytes (coalesced
//     32-bit loads), finds stuffed zeros (FF 00 -> FF) and the terminating marker with byte tests, resolves every
//     kept byte's destination with warp ballots + population-count prefix sums, stages the compacted bytes in shared
//     memory and writes them out as big-endian 32-bit words (coalesced).  What the reference's Fill() does byte by
//     byte (io/bitstream.cpp:56-118) is done here once, in parallel, so the decoder reads plain words.
//
// a1  entropy_decode_kernel -- a warp decodes 32 restart intervals, one per lane, in lock step block by block;
//     persistent CTAs (one per SM, 24 warps) walk the groups of 32 intervals.  Every lane keeps its bit position and
//     the three stream words around it in registers, fed from a 64-byte shared-memory ring that cp.async (LDGSTS,
//     16-byte chunks, topped up at block boundaries, two to four chunks ahead of the reader) keeps filled, so HBM
//     latency never sits on the decode chain.  The scan's Huffman tables live in shared memory as combined
//     (total bits | zig-zag step | code length | value bits) entries; each coefficient is de-zigzagged and
//     dequantised with one more shared-memory lookup and scattered into the lane's 128-byte shared-memory block.
//     At the block boundary the warp stores its 32 blocks together, four complete 128-byte lines per instruction --
//     explicit zeros included, so the coefficient store needs no memset and every line is written exactly once.
//     Warp votes keep the per-symbol loop convergent.  All intervals of all frames that share scan geometry and
//     tables form one launch.
#include <cuda_runtime.h>

#include <cstdint>

#include "internal.hpp"
#include "specsync.hpp"

namespace b200jpg {
namespace {

#ifndef B200JPG_A1_THREADS
#define B200JPG_A1_THREADS 768
#endif
constexpr int kThreads = B200JPG_A1_THREADS;  // a1: CTA size (experiments may override at build time)
constexpr int kStageStride = 144;  // bytes per lane: 128 + 16 pad -> conflict-free 16-byte accesses
constexpr unsigned kFull = 0xffffffffu;

// error codes written to frame_status (reference's numeric values, interface/parameters.hpp:1156-1228)
constexpr uint32_t kErrMalformed = 1038u;      // -(-1038) MALFORMED_STREAM
constexpr uint32_t kErrUnexpectedEof = 1025u;  // -(-1025) UNEXPECTED_EOF

// ---- shared-memory accessors on 32-bit shared-space addresses (keeps the compiler away from generic pointers)
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {  // read-only tables: may be scheduled freely
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ uint32_t lds_u32_v(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts_u16(uint32_t a, int v) { asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "h"((short)v) : "memory"); }
__device__ __forceinline__ void sts_u8(uint32_t a, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ uint4 lds_v4(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_u64(uint32_t a, uint64_t v) { asm volatile("st.shared.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }
__device__ __forceinline__ uint64_t lds_u64(uint32_t a) {
    uint64_t v;
    asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_v4_zero(uint32_t a) {
    asm volatile("st.shared.v4.u32 [%0], {%1,%1,%1,%1};" ::"r"(a), "r"(0u) : "memory");
}
// Integer work that the multiply-add pipe can do is routed there explicitly: the decode loop is bound by the ALU pipe
// (shifts, logic, compares), which takes a warp instruction every other cycle, while the IMAD pipe idles.
__device__ __forceinline__ uint32_t mulhi_u32(uint32_t a, uint32_t b) {
    uint32_t d;
    asm("mul.hi.u32 %0, %1, %2;" : "=r"(d) : "r"(a), "r"(b));
    return d;
}
__device__ __forceinline__ uint32_t mad_u32(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ uint32_t xnor_u32(uint32_t a, uint32_t b) {
    uint32_t d;
    asm("lop3.b32 %0, %1, %2, 0, 0xC3;" : "=r"(d) : "r"(a), "r"(b));
    return d;
}
__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const uint8_t *gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// =====================================================================================================
// a0: byte unstuffing, one warp per restart interval
// =====================================================================================================
constexpr int kUnstuffWarps = 4;

__global__ void __launch_bounds__(kUnstuffWarps * 32)
unstuff_kernel(uint32_t n_intervals, const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ interval_off,
               const uint64_t *__restrict__ interval_end, const uint64_t *__restrict__ clean_off, uint8_t *__restrict__ clean,
               uint32_t *__restrict__ interval_len) {
    __shared__ __align__(16) uint8_t sbuf[kUnstuffWarps][256];
    const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const uint32_t g = blockIdx.x * kUnstuffWarps + wib;
    if (g >= n_intervals) return;  // whole warp
    const uint64_t src0 = interval_off[g];
    if (src0 == ~0ull) {  // interval not present in the stream
        if (lane == 0) interval_len[g] = kIntervalLenAbsent;
        return;
    }
    const uint64_t src1_raw = interval_end[g];
    const uint64_t src1 = src1_raw & ~kIntervalEofFlag;  // offset of the marker (or the end of the data) that ends the interval
    const uint32_t eof_flag = (src1_raw & kIntervalEofFlag) ? kIntervalLenEofFlag : 0u;
    uint32_t *dst = reinterpret_cast<uint32_t *>(clean + clean_off[g]);
    const uint32_t sb = (uint32_t)__cvta_generic_to_shared(&sbuf[wib][0]);
    const uint32_t lt_mask = (1u << lane) - 1u;

    uint32_t fill = 0;     // bytes waiting in sbuf (< 128 between steps)
    uint32_t written = 0;  // words already written to dst
    uint32_t total = 0;    // clean bytes so far
    uint32_t carry_ff = 0; // the last byte of the previous step was a data 0xFF
    bool done = false;
    // the source is read in aligned 32-bit words; bytes in front of src0 are masked out
    for (uint64_t base = src0 & ~3ull; base < src1 && !done; base += 128) {
        const uint64_t wo = base + 4ull * lane;
        uint32_t cur = 0, nxt = 0;
        if (wo < src1) cur = __ldg(reinterpret_cast<const uint32_t *>(bytes + wo));
        if (wo + 4 < src1 + 2) nxt = __ldg(reinterpret_cast<const uint32_t *>(bytes + wo + 4));  // reaches the marker bytes
        // fast path (about 60 % of the steps): no 0xFF anywhere in these 128 bytes and all of them inside the interval:
        // nothing to remove, nothing ends -- the bytes just move
        if (base >= src0 && base + 128 <= src1 && carry_ff == 0 && !__any_sync(kFull, __vcmpeq4(cur, 0xffffffffu) != 0u)) {
            const uint32_t o = fill + 4 * lane;
            if ((fill & 3u) == 0u) {
                sts_u32(sb + o, __byte_perm(cur, 0, 0x0123));
            } else {
#pragma unroll
                for (int k = 0; k < 4; k++) sts_u8(sb + ((o + k) ^ 3u), (cur >> (8 * k)) & 0xffu);
            }
            fill += 128;
            total += 128;
            __syncwarp();
            const uint32_t w = lds_u32_v(sb + 4 * lane);
            const uint32_t w2 = lds_u32_v(sb + 128 + 4 * lane);
            dst[written + lane] = w;
            __syncwarp();
            sts_u32(sb + 4 * lane, w2);
            written += 32;
            fill -= 128;
            __syncwarp();
            continue;
        }
        // byte in front of this lane's word: the previous lane's last byte (lane 0: carried from the last step)
        uint32_t prev_word = __shfl_up_sync(kFull, cur, 1);
        uint32_t keep[4];
        uint32_t mk = 4;  // index of the first marker byte in this word, 4 = none
        // steps that lie inside the interval with room to spare need none of the per-byte range tests
        if (base >= src0 + 4 && base + 132 <= src1) {
            uint32_t pb = (lane == 0) ? (carry_ff ? 0xffu : 0u) : (prev_word >> 24);
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const uint32_t v = (cur >> (8 * k)) & 0xffu;
                const uint32_t nb = (k < 3) ? ((cur >> (8 * k + 8)) & 0xffu) : (nxt & 0xffu);
                if (v == 0xffu && nb != 0u && mk == 4) mk = k;        // FF followed by non-zero (:96-101)
                keep[k] = (v == 0u && pb == 0xffu) ? 0u : 1u;         // the 00 of FF 00 (io/bitstream.cpp:87-95)
                pb = v;
            }
        } else {
            uint32_t pb = (lane == 0) ? (carry_ff ? 0xffu : 0u) : ((wo - 1 >= src0) ? (prev_word >> 24) : 0u);
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const uint64_t q = wo + k;
                const uint32_t v = (cur >> (8 * k)) & 0xffu;
                const uint32_t nb = (k < 3) ? ((cur >> (8 * k + 8)) & 0xffu) : (nxt & 0xffu);
                const bool in = (q >= src0) && (q < src1);
                const bool stuffed = (v == 0u) && (pb == 0xffu);      // the 00 of FF 00 (io/bitstream.cpp:87-95)
                const bool marker = in && (v == 0xffu) && (nb != 0u);  // FF followed by non-zero (:96-101)
                if (marker && mk == 4) mk = k;
                keep[k] = (in && !stuffed) ? 1u : 0u;
                pb = in ? v : 0u;
            }
        }
        // the first lane that holds a marker byte ends the interval: nothing at or after it is data
        const uint32_t mmask = __ballot_sync(kFull, mk < 4);
        const uint32_t first = mmask ? (uint32_t)(__ffs(mmask) - 1) : 32u;
        if (mmask) {
#pragma unroll
            for (int k = 0; k < 4; k++)
                if (lane > first || (lane == first && k >= (int)mk)) keep[k] = 0;
        }
        // destination of every kept byte: one ballot per byte column + population-count prefix sums
        const uint32_t b0 = __ballot_sync(kFull, keep[0]), b1 = __ballot_sync(kFull, keep[1]);
        const uint32_t b2 = __ballot_sync(kFull, keep[2]), b3 = __ballot_sync(kFull, keep[3]);
        const uint32_t before = __popc(b0 & lt_mask) + __popc(b1 & lt_mask) + __popc(b2 & lt_mask) + __popc(b3 & lt_mask);
        const uint32_t step_total = __popc(b0) + __popc(b1) + __popc(b2) + __popc(b3);
        uint32_t o = fill + before;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (keep[k]) {
                sts_u8(sb + (o ^ 3u), (cur >> (8 * k)) & 0xffu);  // ^3: big-endian inside each 32-bit word
                o++;
            }
        }
        carry_ff = __shfl_sync(kFull, ((cur >> 24) == 0xffu && keep[3]) ? 1u : 0u, 31);
        fill += step_total;
        total += step_total;
        done = (first < 32);
        __syncwarp();
        if (fill >= 128) {  // flush 32 complete words, move the rest down
            const uint32_t w = lds_u32_v(sb + 4 * lane);
            const uint32_t w2 = lds_u32_v(sb + 128 + 4 * lane);
            dst[written + lane] = w;
            __syncwarp();
            sts_u32(sb + 4 * lane, w2);
            written += 32;
            fill -= 128;
            __syncwarp();
        }
    }
    // tail: remaining bytes, zero padded to 16 bytes, plus 32 zero bytes so that the decoder reads zeros past the
    // end (the reference feeds zero bits once it stands in front of a marker, io/bitstream.cpp:96-101)
    __syncwarp();
    {
        uint32_t w = lds_u32_v(sb + 4 * lane);
        const uint32_t nbytes = fill, wi = 4 * lane;
        if (wi >= nbytes) w = 0;
        else if (wi + 4 > nbytes) w &= ~0u << (8 * (wi + 4 - nbytes));  // big-endian word: keep the leading bytes
        const uint32_t nwords = (nbytes + 3) / 4;
        const uint32_t padded = ((nwords + 3) & ~3u) + 8;
        if (lane < padded) dst[written + lane] = w;
        if (lane + 32 < padded) dst[written + 32 + lane] = 0;
    }
    if (lane == 0) interval_len[g] = total | eof_flag;
}

// =====================================================================================================
// a0 for restart-less scans: one CTA per interval
// =====================================================================================================
// The whole entropy coded segment of a frame is ONE interval when the stream has no restart markers (megabytes at 4K): a
// single warp walking it would take longer than everything else together. Here the 32 warps of a CTA split it into 32
// byte ranges and run the classification twice -- once to count the bytes every range keeps (and to find the first
// "marker" inside the data, which ends it for the bit reader: io/bitstream.cpp:96-101), then, after a prefix sum over the 32
// counts, to put every kept byte where it belongs. The second pass stores single bytes (at i ^ 3: big-endian words, like the
// warp-per-interval kernel writes them): a warp's bytes are consecutive, so they coalesce, and nothing has to be merged
// where two ranges meet in the middle of a word.
constexpr int kLongThreads = 1024;

#ifndef B200JPG_LONG_MINCTAS
#define B200JPG_LONG_MINCTAS 2
#endif
__global__ void __launch_bounds__(kLongThreads, B200JPG_LONG_MINCTAS)
unstuff_long_kernel(uint32_t n_intervals, const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ interval_off,
                    const uint64_t *__restrict__ interval_end, const uint64_t *__restrict__ clean_off, uint8_t *__restrict__ clean,
                    uint32_t *__restrict__ interval_len) {
    __shared__ uint32_t s_count[32];
    __shared__ unsigned long long s_marker;  // offset of the first FF xx (xx != 0) inside the data, ~0 = none
    const uint32_t g = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (g >= n_intervals) return;
    const uint64_t src0 = interval_off[g];
    if (src0 == ~0ull) {
        if (threadIdx.x == 0) interval_len[g] = kIntervalLenAbsent;
        return;
    }
    const uint64_t src1_raw = interval_end[g];
    const uint64_t src1 = src1_raw & ~kIntervalEofFlag;
    const uint32_t eof_flag = (src1_raw & kIntervalEofFlag) ? kIntervalLenEofFlag : 0u;
    if (threadIdx.x == 0) s_marker = ~0ull;
    __syncthreads();
    // byte ranges of the warps: multiples of 128 bytes counted from the aligned start
    const uint64_t base0 = src0 & ~3ull;
    const uint64_t steps = (src1 - base0 + 127) / 128;
    const uint64_t per = (steps + 31) / 32;
    const uint64_t lo = base0 + 128 * per * warp;
    uint64_t hi = lo + 128 * per;
    if (hi > src1) hi = src1;
    uint8_t *dst = clean + clean_off[g];
    // one step of 128 bytes: keep[k] = byte k of this lane's word is data; returns the number of bytes the warp keeps
    auto classify = [&](uint64_t base, uint64_t limit, uint32_t &cur, uint32_t (&keep)[4]) -> uint32_t {
        const uint64_t wo = base + 4ull * lane;
        cur = 0;
        uint32_t nxt = 0, prv = 0;
        if (wo < src1) cur = __ldg(reinterpret_cast<const uint32_t *>(bytes + wo));
        if (wo + 4 < src1 + 2) nxt = __ldg(reinterpret_cast<const uint32_t *>(bytes + wo + 4));
        if (wo >= src0 + 1) prv = bytes[wo - 1];
        uint32_t pb = prv, n = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint64_t q = wo + k;
            const uint32_t v = (cur >> (8 * k)) & 0xffu;
            const uint32_t nb = (k < 3) ? ((cur >> (8 * k + 8)) & 0xffu) : (nxt & 0xffu);
            const bool in = q >= src0 && q < limit;
            if (in && v == 0xffu && nb != 0u) atomicMin(&s_marker, (unsigned long long)q);  // rare: data that runs into a marker
            keep[k] = (in && !(v == 0u && pb == 0xffu && q > src0)) ? 1u : 0u;  // the 00 of FF 00 goes (io/bitstream.cpp:87-95)
            n += keep[k];
            pb = v;
        }
        return n;
    };
    // steps that lie inside this warp's range with room to spare and hold no 0xFF at all (about 60 % of them) keep every byte
    auto plain_step = [&](uint64_t base, uint64_t limit, uint32_t &cur) -> bool {
        if (base < src0 + 4 || base + 132 > limit) return false;  // (warp-uniform)
        cur = __ldg(reinterpret_cast<const uint32_t *>(bytes + base + 4ull * lane));
        const uint32_t prv = (lane == 0) ? bytes[base - 1] : 0u;   // a 00 at the front of the step could follow an FF of the last one
        return !__any_sync(kFull, __vcmpeq4(cur, 0xffffffffu) != 0u || prv == 0xffu);
    };
    // ---- pass 1: count
    uint32_t mine = 0;
    for (uint64_t base = lo; base < hi; base += 128) {
        uint32_t cur, keep[4];
        if (plain_step(base, hi, cur)) mine += 4;
        else mine += classify(base, hi, cur, keep);
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) mine += __shfl_xor_sync(kFull, mine, d);
    if (lane == 0) s_count[warp] = mine;
    __syncthreads();
    const uint64_t marker = s_marker;
    if (marker != ~0ull) {
        // a marker inside the data: everything from it on is not data. Recount with the ranges clipped (rare path).
        const uint64_t lim = hi < marker ? hi : marker;
        mine = 0;
        for (uint64_t base = lo; base < lim; base += 128) {
            uint32_t cur, keep[4];
            mine += classify(base, lim, cur, keep);
        }
#pragma unroll
        for (int d = 16; d; d >>= 1) mine += __shfl_xor_sync(kFull, mine, d);
        __syncthreads();
        if (lane == 0) s_count[warp] = mine;
        __syncthreads();
        if (hi > marker) hi = marker;
    }
    uint32_t before = 0, total = 0;
    for (int i = 0; i < 32; i++) {
        const uint32_t c = s_count[i];
        if (i < (int)warp) before += c;
        total += c;
    }
    // ---- pass 2: place
    const uint32_t lt_mask = (1u << lane) - 1u;
    uint32_t out = before;
    for (uint64_t base = lo; base < hi; base += 128) {
        uint32_t cur, keep[4];
        if (plain_step(base, hi, cur)) {  // 128 bytes move as they are: one word store per lane when the destination is aligned
            const uint32_t o = out + 4u * lane;
            if ((out & 3u) == 0u) {
                *reinterpret_cast<uint32_t *>(dst + o) = __byte_perm(cur, 0, 0x0123);
            } else {
#pragma unroll
                for (int k = 0; k < 4; k++) dst[(o + k) ^ 3u] = (uint8_t)(cur >> (8 * k));
            }
            out += 128;
            continue;
        }
        classify(base, hi, cur, keep);
        const uint32_t b0 = __ballot_sync(kFull, keep[0]), b1 = __ballot_sync(kFull, keep[1]);
        const uint32_t b2 = __ballot_sync(kFull, keep[2]), b3 = __ballot_sync(kFull, keep[3]);
        uint32_t o = out + __popc(b0 & lt_mask) + __popc(b1 & lt_mask) + __popc(b2 & lt_mask) + __popc(b3 & lt_mask);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (keep[k]) {
                dst[o ^ 3u] = (uint8_t)(cur >> (8 * k));
                o++;
            }
        }
        out += __popc(b0) + __popc(b1) + __popc(b2) + __popc(b3);
    }
    // ---- tail: zero up to the next 16-byte boundary + 32 bytes (the decoder reads zeros behind the data, :96-105)
    const uint32_t end_pad = ((total + 15u) & ~15u) + 32u;
    for (uint32_t i = total + threadIdx.x; i < end_pad; i += kLongThreads) dst[i ^ 3u] = 0;
    if (threadIdx.x == 0) interval_len[g] = total | eof_flag;
}

// =====================================================================================================
// a1: Huffman decode, one restart interval per lane
// =====================================================================================================
// B200JPG_A1_PACKED_PAIR: the (q, byte offset) pair of a zig-zag position as ONE word in shared memory, q << 8 | offset
// (q < 2^24, parse.cpp; offsets <= 128): a 4-byte load per symbol is one L1 wavefront before bank conflicts, the 8-byte load of
// the table's global form two. B200JPG_A1_SHFL_DST: the flush learns where the other lanes' blocks go by shuffle (a 32-bit
// block number) instead of through the pad of the staging blocks (an 8-byte shared load per lane and step).
#ifndef B200JPG_A1_PACKED_PAIR
#define B200JPG_A1_PACKED_PAIR 1
#endif
#ifndef B200JPG_A1_SHFL_DST
#define B200JPG_A1_SHFL_DST 1
#endif
constexpr int kQzPairBytes = B200JPG_A1_PACKED_PAIR ? 4 : 8;
constexpr int kQzBytes = 4 * kQzEntries * kQzPairBytes;  // four quantisation tables of (q, offset) pairs
constexpr int kBdescBytes = 16 * 16;          // indexed decoding: one 16-byte descriptor per block of an MCU (at most 10)

// kIndexed: the work items are the SpecSegments that spec_sync_kernel cut out of restart-less scans (specsync.hpp) instead of
// restart intervals: a lane starts at any bit, at any block of an MCU, with the DC predictors of that place, and decodes a
// number of blocks; everything per block -- tables, quantiser, destination -- is then a per-lane quantity (a small table in
// shared memory indexed by the block's position in its MCU), while the symbol decoder, the ring and the flush are the same.
template <bool kLutShared, bool kIndexed>
__global__ void __launch_bounds__(kThreads, 1)
entropy_decode_kernel(ScanClassParams p, const uint8_t *__restrict__ clean, const uint64_t *__restrict__ clean_off,
                      const uint32_t *__restrict__ interval_len, const ClassScan *__restrict__ scans,
                      const uint8_t *__restrict__ tables, int16_t *__restrict__ coef, uint32_t *__restrict__ frame_status,
                      uint32_t *__restrict__ overrun_list, const SpecSegment *__restrict__ segments) {
    extern __shared__ __align__(16) uint8_t smem[];
    // layout (bytes): [stage: kThreads*144][ring: kThreads*64][qz: 4*128*8][lut: lut_words*4 (if shared)]
    uint32_t s_base = (uint32_t)__cvta_generic_to_shared(smem);
    asm volatile("" : "+r"(s_base));  // opaque: keeps the base in a register instead of re-deriving it (S2UR) at every use
    const uint32_t s_stage = s_base + threadIdx.x * kStageStride;
    const uint32_t s_ring = s_base + kThreads * kStageStride + threadIdx.x * 64;
    const uint32_t s_qz = s_base + kThreads * kStageStride + kThreads * 64;
    const uint32_t s_bdesc = s_qz + kQzBytes;  // kIndexed: per block of an MCU {DC table, AC table, quantiser pairs, c | x << 8 | y << 16}
    const uint32_t s_lut = s_bdesc + (kIndexed ? kBdescBytes : 0);
    // cooperative flush: in step i this lane moves bytes [16*(lane&7), +16) of the block staged by lane 4*i + (lane>>3)
    const uint32_t s_flush_sub = (threadIdx.x & 7u) << 4;
    const uint32_t s_flush = s_base + ((threadIdx.x & ~31u) + ((threadIdx.x & 31u) >> 3)) * kStageStride + s_flush_sub;
    const uint32_t *g_lut = reinterpret_cast<const uint32_t *>(tables + kTableHeaderBytes);
    {
        const uint32_t *g_qz = reinterpret_cast<const uint32_t *>(tables + 32);
#if B200JPG_A1_PACKED_PAIR
        for (uint32_t i = threadIdx.x; i < 4 * kQzEntries; i += kThreads) sts_u32(s_qz + 4 * i, (g_qz[2 * i] << 8) | g_qz[2 * i + 1]);
#else
        for (uint32_t i = threadIdx.x; i < kQzBytes / 4; i += kThreads) sts_u32(s_qz + 4 * i, g_qz[i]);
#endif
        if (kLutShared)
            for (uint32_t i = threadIdx.x; i < p.lut_words; i += kThreads) sts_u32(s_lut + 4 * i, g_lut[i]);
#pragma unroll
        for (int i = 0; i < 9; i++) sts_v4_zero(s_stage + 16 * i);
    }
    __syncthreads();
    const uint16_t *lut_off = reinterpret_cast<const uint16_t *>(tables + 16);

    // Persistent CTAs (one per SM): warp w of CTA b takes the groups of 32 consecutive restart intervals b + gridDim.x * w,
    // then every (gridDim.x * warps per CTA)-th one after that, so any batch size spreads evenly over the SMs.
    const uint64_t total_intervals = (uint64_t)p.n_scans * (kIndexed ? p.segs_per_scan : p.intervals_per_scan);
    const uint64_t n_groups = (total_intervals + 31u) / 32u;
    if (kIndexed) {
        if (threadIdx.x == 0) {
            uint32_t b = 0;
            for (int c = 0; c < p.ns; c++)
                for (int y = 0; y < p.mh[c]; y++)
                    for (int x = 0; x < p.mw[c]; x++, b++) {
                        sts_u32(s_bdesc + 16 * b, s_lut + 4u * lut_off[p.dc_slot[c]]);
                        sts_u32(s_bdesc + 16 * b + 4, s_lut + 4u * lut_off[4 + p.ac_slot[c]]);
                        sts_u32(s_bdesc + 16 * b + 8, s_qz + (uint32_t)(kQzEntries * kQzPairBytes) * p.q_slot[c]);
                        sts_u32(s_bdesc + 16 * b + 12, (uint32_t)c | ((uint32_t)x << 8) | ((uint32_t)y << 16));
                    }
        }
        __syncthreads();
    }
    for (uint64_t grp = blockIdx.x + (uint64_t)gridDim.x * (threadIdx.x >> 5); grp < n_groups; grp += (uint64_t)gridDim.x * (kThreads / 32)) {
        const uint64_t g = grp * 32u + (threadIdx.x & 31u);
        cp_async_wait<0>();  // nothing of the previous group may still land in the ring
        const bool lane_valid = g < total_intervals;
        uint32_t j = 0, iv = 0;
        if (lane_valid) {
            j = (uint32_t)(g / (kIndexed ? p.segs_per_scan : p.intervals_per_scan));
            iv = (uint32_t)(g % (kIndexed ? p.segs_per_scan : p.intervals_per_scan));
        }
        // indexed: the scan is ONE unstuffed interval (number j); this lane's work item starts seg_bit bits into it
        uint32_t seg_bit = 0, seg_first = 0, seg_blocks = 0;
        int seg_pred[4] = {0, 0, 0, 0};
        if (kIndexed && lane_valid) {
            const uint4 a = __ldg(reinterpret_cast<const uint4 *>(segments + g));
            const uint4 b = __ldg(reinterpret_cast<const uint4 *>(segments + g) + 1);
            seg_bit = a.x, seg_first = a.y, seg_blocks = a.z;
            seg_pred[0] = (int)a.w, seg_pred[1] = (int)b.x, seg_pred[2] = (int)b.y, seg_pred[3] = (int)b.z;
        }
        const uint32_t len_raw = lane_valid ? interval_len[kIndexed ? (uint64_t)j : g] : 0u;
        const uint32_t seg_skip = (seg_bit >> 7) << 4;  // whole 16-byte chunks in front of the work item
        const uint32_t len_all = len_raw & kIntervalLenMask;
        const uint32_t len_bytes = kIndexed ? (len_all > seg_skip ? len_all - seg_skip : 0u) : len_all;
        const uint8_t *src = clean + (lane_valid ? clean_off[kIndexed ? (uint64_t)j : g] : 0ull) + seg_skip;
        const uint32_t max_chunks = (len_bytes + 15u) / 16u + 2u;  // data + the 32 zero bytes a0 appended
        const uint32_t mcu0 = kIndexed ? seg_first / (uint32_t)(p.mw[0] * p.mh[0] + (p.ns > 1 ? p.mw[1] * p.mh[1] : 0) + (p.ns > 2 ? p.mw[2] * p.mh[2] : 0) +
                                                                (p.ns > 3 ? p.mw[3] * p.mh[3] : 0))
                                       : iv * p.dri;
        uint32_t nmcu = 0;
        if (lane_valid) nmcu = (p.total_mcus - mcu0 < p.dri) ? (p.total_mcus - mcu0) : p.dri;
        uint32_t mx = mcu0 % p.mcu_cols, my = mcu0 / p.mcu_cols;

        uint64_t plane[4];
        uint32_t frame = 0;
        {
            const ClassScan &cs = scans[lane_valid ? j : 0];
#pragma unroll
            for (int c = 0; c < 4; c++) plane[c] = cs.coef_base[c];
            frame = cs.frame;
        }

        // an interval the stream does not contain keeps its blocks zero (sequentialscan.cpp:415-419)
        const bool decoding = lane_valid && !(len_raw & kIntervalLenAbsent) && (!kIndexed || seg_blocks != 0u);
        // Bit reader. bp = bits consumed so far; x0, x1, x2 = the stream words bp/32, +1 and +2 (x2 is a prefetch, so the
        // shared-memory latency of the ring never sits on the decode chain). The 32 bits at bp are one funnel shift of
        // (x0, x1); consuming bits is an addition, and when bp enters the next word the three registers move up by one.
        // req = 16-byte chunks requested from HBM so far, safe_w = stream words known to have landed in the ring.
        uint32_t bp = kIndexed ? (seg_bit & 127u) : 0u, xw = bp >> 5, x0 = 0, x1 = 0, x2 = 0, req = 0, safe_w = 0;
        // chunk `c` of the interval into its ring slot; past the end of the interval the reader sees zeros, exactly what
        // the reference's bit reader hands out once it stands in front of a marker (io/bitstream.cpp:96-101)
        auto request = [&](uint32_t c) {
            if (c < max_chunks) cp_async16(s_ring + ((c & 3u) << 4), src + ((uint64_t)c << 4));
            else sts_v4_zero(s_ring + ((c & 3u) << 4));
        };
        if (decoding) {
#pragma unroll
            for (uint32_t i = 0; i < 4; i++) request(i);
            req = 4;
        }
        cp_async_commit();
        cp_async_wait<0>();
        safe_w = req << 2;
        if (decoding) {
            x0 = lds_u32_v(s_ring + 4 * xw);
            x1 = lds_u32_v(s_ring + 4 * xw + 4);
            x2 = lds_u32_v(s_ring + 4 * xw + 8);
        }

        uint32_t errbits = 0;  // bit 31: an entry that must not be decoded was decoded
        uint32_t ovf = 0;      // | (v + 32768): bits 16.. set when a dequantised coefficient left the int16 range
        int pred[4] = {seg_pred[0], seg_pred[1], seg_pred[2], seg_pred[3]};
        uint32_t dc_off[4], ac_off[4], q_addr[4];
#pragma unroll
        for (int c = 0; c < 4; c++) {
            dc_off[c] = (c < p.ns) ? s_lut + 4u * lut_off[p.dc_slot[c]] : 0;
            ac_off[c] = (c < p.ns) ? s_lut + 4u * lut_off[4 + p.ac_slot[c]] : 0;
            q_addr[c] = s_qz + ((c < p.ns) ? (uint32_t)(kQzEntries * kQzPairBytes) * p.q_slot[c] : 0u);
        }

        // A symbol has fewer than 32 bits, so bp crosses at most one word boundary. The moves and the load of the new x2
        // are predicated: lanes that stay inside their word keep their registers, and no move waits for the load.
        auto advance = [&](uint32_t e) {
            bp += e >> 26;  // total bits of the symbol (error entries: + 32, the lane stops anyway)
            const uint32_t w = bp >> 5, nw = w + 2u;
            if (nw >= safe_w) {  // rare: about to run past what the block-boundary top-up guarantees
                while (req <= (nw >> 2)) request(req++);
                cp_async_commit();
                cp_async_wait<0>();
                safe_w = req << 2;
            }
            const uint32_t c = w - xw;  // 0 or 1
            x0 = mad_u32(c, x1 - x0, x0);
            x1 = mad_u32(c, x2 - x1, x1);
            asm volatile("{ .reg .pred c; setp.ne.u32 c, %1, 0; @c ld.shared.u32 %0, [%2]; }"
                         : "+r"(x2)
                         : "r"(c), "r"(s_ring + (mad_u32(nw, 4u, 0u) & 0x3cu))
                         : "memory");
            xw = w;
        };
        // two-level lookup in the window `hi`; `tab` is the shared-space address of the table (kLutShared) or stands for
        // its word offset (global). Codes longer than kLutL1Bits are rare.
        auto lookup = [&](uint32_t tab, uint32_t hi) -> uint32_t {
            constexpr uint32_t kSubMask = (1u << (16 - kLutL1Bits)) - 1u;
            uint32_t e;
            if (kLutShared) {
                e = lds_u32(mad_u32(mulhi_u32(hi, 1u << kLutL1Bits), 4u, tab));
                if ((e & (31u << 5)) == 0) e = lds_u32(tab + (((1u << kLutL1Bits) + ((e >> 10) << (16 - kLutL1Bits)) + ((hi >> 16) & kSubMask)) << 2));
            } else {
                const uint32_t *t = g_lut + ((tab - s_lut) >> 2);
                e = __ldg(t + (hi >> (32 - kLutL1Bits)));
                if ((e & (31u << 5)) == 0) e = __ldg(t + (1u << kLutL1Bits) + ((e >> 10) << (16 - kLutL1Bits)) + ((hi >> 16) & kSubMask));
            }
            return e;
        };
        // value bits of entry e, sign-extended as sequentialscan.cpp:692-696 / 757-762: first value bit set = the bits
        // are the value, otherwise their complement is the magnitude of a negative value. All shifts are funnel shifts in
        // wrap mode, which use only the low five bits of the count: the fields of e need no masking.
        auto value_of = [&](uint32_t e, uint32_t hi) -> int {
            const uint32_t t = __funnelshift_l(0u, hi, e >> 5);   // hi << len: value bits at the top
            const int pos = (int)t >> 31;                         // -1: non-negative value, 0: negative
            const uint32_t mag = __funnelshift_l(xnor_u32(t, (uint32_t)pos), 0u, e);  // >> (32 - s); 0 for s == 0
            return (int)mag * (-2 * pos - 1);
        };

        // ---- one block: `has` says whether this lane has a block in this step; tables, predictor and destination are the
        // caller's (warp-uniform compile-time choices for restart intervals, per-lane values for indexed work items)
        auto decode_block = [&](const bool has, const uint32_t dc_tab, const uint32_t ac_tab, const uint32_t q_tab, int &predc, const int16_t *d) {
            // ---- convergent ring top-up: keep the reader two to four 16-byte chunks ahead
            {
                const uint32_t ch = bp >> 7;
                const uint32_t landed = req;  // requested before this point: lands at the wait below
#pragma unroll
                for (int t = 0; t < 2; t++) {
                    if (decoding && req < ch + 4u) request(req++);
                    cp_async_commit();
                }
                cp_async_wait<2>();
                safe_w = landed << 2;
            }
            // a lane that met an error keeps its blocks zero from there on. k = zig-zag index of the next
            // coefficient; k > 63: the lane has nothing (more) to decode in this block
            int k = 64;
            // The dequantise + store of a coefficient is deferred by one symbol: its table pair (pq) is loaded
            // when the symbol is decoded and consumed after the NEXT symbol's table lookup has been issued, so
            // neither shared-memory latency is exposed. {0, 128} parks a "nothing pending" store in the pad slot.
            uint2 pq = make_uint2(B200JPG_A1_PACKED_PAIR ? 128u : 0u, 128u);
            int pd = 0;
            auto load_pair = [&](uint32_t k_minus_1_scaled_addr) {
#if B200JPG_A1_PACKED_PAIR
                pq.x = lds_u32(k_minus_1_scaled_addr);  // unpacked where it is consumed (drain), not behind the load
#else
                asm("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(pq.x), "=r"(pq.y) : "r"(k_minus_1_scaled_addr));
#endif
            };
            auto drain = [&]() {
#if B200JPG_A1_PACKED_PAIR
                const uint32_t q = pq.x >> 8, off = pq.x & 0xffu;
#else
                const uint32_t q = pq.x, off = pq.y;
#endif
                const int v = pd * (int)q;
                ovf |= mad_u32((uint32_t)pd, q, 32768u);
                sts_u16(s_stage + off, v);
            };
            // ---- DC: sequentialscan.cpp:682-701
            if (has && decoding && (int)errbits >= 0) {
                const uint32_t hi = __funnelshift_l(x1, x0, bp);
                const uint32_t e = lookup(dc_tab, hi);
                errbits |= e;
                if ((int)e >= 0) {
                    predc += value_of(e, hi);
                    advance(e);
                    pd = predc;
                    load_pair(q_tab);
                    k = 1;
                }
            }
            // ---- AC: sequentialscan.cpp:704-771, one symbol per warp-convergent iteration. The table entry
            // carries the step of the zig-zag index: run + 1 for a coefficient, 16 for ZRL (the reference
            // re-tests k <= 63 and silently ends the block, :717-719), kQzBlockEnds for EOB and for entries
            // that must not be decoded (bit 31). The table pair is fetched at k - 1 in every case: symbols
            // without value bits store a zero (ZRL: in a position that is zero anyway; block end: pad slot),
            // a coefficient whose run leaves the block hits a pair that multiplies it out of the int16 range
            // (:764-766: out of sync), a ZRL that leaves it multiplies its zero and just ends the block.
            while (__any_sync(kFull, k <= 63)) {
                if (k <= 63) {
                    const uint32_t hi = __funnelshift_l(x1, x0, bp);
                    const uint32_t e = lookup(ac_tab, hi);
                    drain();
                    errbits |= e;
                    pd = value_of(e, hi);  // 0 when the symbol carries no value bits
                    advance(e);
                    k += (int)mulhi_u32(mad_u32(e, 64u, 0u), 128u);  // bits 25:19
                    load_pair(mad_u32((uint32_t)k, (uint32_t)kQzPairBytes, q_tab - (uint32_t)kQzPairBytes));
                }
            }
            drain();
            // ---- flush (zeros included) and clear the staging blocks, the whole warp together: every lane
            // publishes where its block goes (0 = nowhere) in the pad of its staging block, then each store
            // instruction moves four complete 128-byte blocks (eight lanes x 16 bytes per block) instead of one
            // 16-byte piece of 32 different blocks -- 4 instead of 32 L1 wavefronts per instruction
            {
#if B200JPG_A1_SHFL_DST
                // the block's number in the coefficient store + 1 (0 = nowhere): 32 bits are enough for 2^32 blocks of 128 bytes
                const uint32_t mine = has ? (uint32_t)((d - coef) >> 6) + 1u : 0u;
                __syncwarp();
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    const uint32_t a = s_flush + i * (4 * kStageStride);
                    const uint32_t blk = __shfl_sync(kFull, mine, 4 * i + (int)((threadIdx.x & 31u) >> 3));
                    const uint4 v = lds_v4(a);
                    sts_v4_zero(a);
                    if (blk) *reinterpret_cast<uint4 *>(reinterpret_cast<uint8_t *>(coef) + ((uint64_t)(blk - 1u) << 7) + s_flush_sub) = v;
                }
                __syncwarp();
#else
                sts_u64(s_stage + 136, has ? (uint64_t)d : 0ull);
                __syncwarp();
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    const uint32_t a = s_flush + i * (4 * kStageStride);
                    const uint64_t dst = lds_u64(a + 136 - s_flush_sub);
                    const uint4 v = lds_v4(a);
                    sts_v4_zero(a);
                    if (dst) *reinterpret_cast<uint4 *>(dst + s_flush_sub) = v;
                }
                __syncwarp();
#endif
            }
        };

        if (!kIndexed) {
            for (uint32_t mi = 0; mi < p.dri; mi++) {
                const bool has_mcu = mi < nmcu;
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    if (c >= p.ns) break;
                    for (int y = 0; y < p.mh[c]; y++) {
                        for (int x = 0; x < p.mw[c]; x++) {
                            const uint32_t bx = mx * p.mw[c] + x, by = my * p.mh[c] + y;
                            decode_block(has_mcu, dc_off[c], ac_off[c], q_addr[c], pred[c], coef + plane[c] + ((uint64_t)by * p.bw[c] + bx) * 64u);
                        }
                    }
                }
                if (++mx == p.mcu_cols) {
                    mx = 0;
                    my++;
                }
            }
        } else {
            // per-lane walk over this work item's blocks: block b of MCU (mx, my); the warp runs as long as its longest item
            uint32_t bpm = 0;
            for (int c = 0; c < p.ns; c++) bpm += (uint32_t)(p.mw[c] * p.mh[c]);
            uint32_t b = seg_first % bpm;
            const uint32_t nb = decoding ? seg_blocks : 0u;
            const uint32_t max_nb = __reduce_max_sync(kFull, nb);
            for (uint32_t bi = 0; bi < max_nb; bi++) {
                const bool has = bi < nb;
                const uint4 bd = lds_v4(s_bdesc + 16u * b);
                const uint32_t c = bd.w & 0xffu, x = (bd.w >> 8) & 0xffu, y = bd.w >> 16;
                const uint32_t mw = c == 0 ? (uint32_t)p.mw[0] : (c == 1 ? (uint32_t)p.mw[1] : (c == 2 ? (uint32_t)p.mw[2] : (uint32_t)p.mw[3]));
                const uint32_t mh = c == 0 ? (uint32_t)p.mh[0] : (c == 1 ? (uint32_t)p.mh[1] : (c == 2 ? (uint32_t)p.mh[2] : (uint32_t)p.mh[3]));
                const uint32_t bw = c == 0 ? (uint32_t)p.bw[0] : (c == 1 ? (uint32_t)p.bw[1] : (c == 2 ? (uint32_t)p.bw[2] : (uint32_t)p.bw[3]));
                const uint64_t pl = c == 0 ? plane[0] : (c == 1 ? plane[1] : (c == 2 ? plane[2] : plane[3]));
                int pr = c == 0 ? pred[0] : (c == 1 ? pred[1] : (c == 2 ? pred[2] : pred[3]));
                const uint32_t bx = mx * mw + x, by = my * mh + y;
                decode_block(has, bd.x, bd.y, bd.z, pr, coef + pl + ((uint64_t)by * bw + bx) * 64u);
                pred[0] = c == 0 ? pr : pred[0], pred[1] = c == 1 ? pr : pred[1], pred[2] = c == 2 ? pr : pred[2], pred[3] = c == 3 ? pr : pred[3];
                if (++b == bpm) {
                    b = 0;
                    if (++mx == p.mcu_cols) {
                        mx = 0;
                        my++;
                    }
                }
            }
        }
        uint32_t err = 0;
        if ((int)errbits < 0 || (ovf >> 16) != 0u) {
            err = kErrMalformed;  // invalid code / out-of-sync coefficient index / coefficient beyond the int16 store
        } else if (decoding) {
            // A valid stream never consumes bits beyond the marker that ends its interval. One that does is not necessarily an
            // error to the reference (its bit reader hands out a byte of zero bits per refill in front of a marker and only
            // throws when one request cannot be met, io/bitstream.hpp:168-208): overrun_verdict_kernel decides.
            const uint64_t consumed = bp;
            // (indexed work items: a cut restart-less scan just runs on through zero bits like the reference's reader does)
            if (!kIndexed && consumed > (uint64_t)len_bytes * 8u && !(len_raw & kIntervalLenEofFlag)) overrun_list[1u + atomicAdd(overrun_list, 1u)] = (uint32_t)g;
        }
        if (err) atomicMax(frame_status + frame, err);
    }
}


// =====================================================================================================
// overrun verdict: the intervals whose decoder read past their terminating marker, replayed with the reference's bit reader
// =====================================================================================================
// BitStream<false> (io/bitstream.hpp:168-208, io/bitstream.cpp:56-118) keeps m_ucBits buffered bits. Fill() -- called by
// PeekWord() when fewer than 16 bits are buffered and by Get(n) when fewer than n are -- pulls bytes while at most 24 bits are
// buffered; standing in front of a marker it adds ONE byte of zero bits per call and returns. SkipBits(n) (the code length
// after a PeekWord) and Get(n) (the value bits) throw UNEXPECTED_EOF when, after that, fewer than n bits are buffered. So a
// damaged interval may run on through zero bits for as long as every single request is small -- with the usual tables it
// always does -- and the frame decodes (with whatever those zero bits mean); only this replay knows. One thread per listed
// interval, symbol lengths only; rare by construction (damaged streams), so nothing here is tuned.
__global__ void __launch_bounds__(128)
overrun_verdict_kernel(ScanClassParams p, const uint8_t *__restrict__ clean, const uint64_t *__restrict__ clean_off,
                       const uint32_t *__restrict__ interval_len, const ClassScan *__restrict__ scans, const uint8_t *__restrict__ tables,
                       const uint32_t *__restrict__ list, uint32_t *__restrict__ frame_status) {
    const uint32_t n = list[0];
    const uint32_t *g_lut = reinterpret_cast<const uint32_t *>(tables + kTableHeaderBytes);
    const uint16_t *lut_off = reinterpret_cast<const uint16_t *>(tables + 16);
    for (uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += gridDim.x * blockDim.x) {
        const uint32_t g = list[1 + idx];
        const uint32_t j = g / p.intervals_per_scan, iv = g % p.intervals_per_scan;
        const uint32_t len_bytes = interval_len[g] & kIntervalLenMask;
        const uint32_t *w = reinterpret_cast<const uint32_t *>(clean + clean_off[g]);
        const uint32_t nwords = (len_bytes + 3u) / 4u;
        const uint32_t real = len_bytes * 8u;  // bits in front of the marker
        const uint32_t mcu0 = iv * p.dri;
        const uint32_t nmcu = (p.total_mcus - mcu0 < p.dri) ? (p.total_mcus - mcu0) : p.dri;
        uint32_t bp = 0, loaded = 0;  // bits consumed; bits pulled into the reader's buffer (zero bytes in front of the marker included)
        bool thrown = false, stop = false;
        auto fill = [&]() {
            do {
                const bool at_marker = loaded >= real;
                loaded += 8u;
                if (at_marker) break;
            } while (loaded - bp <= 24u);
        };
        auto window = [&]() -> uint32_t {  // the 32 bits at bp; zero bits behind the data
            const uint32_t i = bp >> 5;
            const uint32_t w0 = i < nwords ? __ldg(w + i) : 0u, w1 = i + 1u < nwords ? __ldg(w + i + 1u) : 0u;
            return __funnelshift_l(w1, w0, bp);
        };
        auto symbol = [&](uint32_t slot) -> uint32_t {  // HuffmanDecoder::Get: PeekWord + SkipBits
            if (loaded - bp < 16u) fill();
            const uint32_t hi = window();
            const uint32_t *t = g_lut + lut_off[slot];
            uint32_t e = __ldg(t + (hi >> (32 - kLutL1Bits)));
            if ((e & (31u << 5)) == 0) e = __ldg(t + (1u << kLutL1Bits) + ((e >> 10) << (16 - kLutL1Bits)) + ((hi >> 16) & ((1u << (16 - kLutL1Bits)) - 1u)));
            if ((int)e < 0) {  // a code the tables do not define: the sequential kernel has reported it already
                stop = true;
                return e;
            }
            const uint32_t len = (e >> 5) & 31u;
            if (len > loaded - bp) thrown = true;
            bp += len;
            return e;
        };
        auto get = [&](uint32_t s) {  // BitStream::Get(s), s >= 1
            if (s > loaded - bp) {
                fill();
                if (s > loaded - bp) thrown = true;
            }
            bp += s;
        };
        for (uint32_t mi = 0; mi < nmcu && !thrown && !stop; mi++)
            for (int c = 0; c < p.ns && !thrown && !stop; c++)
                for (int b = 0; b < p.mw[c] * p.mh[c] && !thrown && !stop; b++) {
                    uint32_t e = symbol((uint32_t)p.dc_slot[c]);
                    if (thrown || stop) break;
                    if (e & 31u) get(e & 31u);
                    int k = 1;
                    while (k <= 63 && !thrown && !stop) {
                        e = symbol(4u + (uint32_t)p.ac_slot[c]);
                        if (thrown || stop) break;
                        const uint32_t s = e & 31u, step = (e >> 19) & 127u;
                        if (s == 0u) {
                            if (step == 16u) {
                                k += 16;  // ZRL
                                continue;
                            }
                            break;  // EOB
                        }
                        k += (int)step - 1;
                        get(s);
                        if (k >= 64) stop = true;  // out of sync: reported by the sequential kernel
                        k++;
                    }
                }
        if (thrown) atomicMax(frame_status + scans[j].frame, kErrUnexpectedEof);
    }
}

// =====================================================================================================
// restart index: one CTA per scan (SURVEY 8f1)
// =====================================================================================================
// What the host parser's walk over the entropy coded segment does with memchr (parse.cpp index_ecs: FF 00 is a
// stuffed byte, FF FF a fill byte in front of a marker, entropyparser.cpp:121-125; RSTn ends an interval; anything
// else ends the segment), byte-parallel: 256 threads test 16 bytes each per step, a block-wide prefix sum numbers the
// restart markers in stream order, and the scan's slices of the interval arrays are written in place:
//   interval k = [off[k], end[k]);  off[0] = ecs_off, off[k+1] = RST_k + 2, end[k] = RST_k (last one: the marker that ends
//   the segment, or a surplus RST);  intervals the stream does not contain: off = ~0 (zero-filled by the decoder);
//   RST_k is expected to be RST(k mod 8); otherwise the reference's resynchronisation (entropyparser.cpp:137-199) is replayed
//   over the marker list by one thread (lost intervals: off = ~0);
//   clean_off[k] = base + (off[k] - ecs_off) + 80 k rounded up to 16: unstuffing never grows the data, so the pieces
//   cannot overlap and no lengths have to be known on the host.
constexpr int kIndexThreads = 256;

__global__ void __launch_bounds__(kIndexThreads)
restart_index_kernel(const IndexScan *__restrict__ scans, uint8_t *__restrict__ input, uint32_t *__restrict__ index_status) {
    const IndexScan s = scans[blockIdx.x];
    uint64_t *off = reinterpret_cast<uint64_t *>(input + s.off_arr);
    uint64_t *end = reinterpret_cast<uint64_t *>(input + s.end_arr);
    uint64_t *cln = reinterpret_cast<uint64_t *>(input + s.clean_arr);
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t nint = s.n_intervals;
    __shared__ uint32_t warp_cnt[kIndexThreads / 32];
    __shared__ unsigned long long first_other;  // lowest offset of a marker that is not RSTn, ~0 = none so far
    if (tid == 0) first_other = ~0ull;
    __syncthreads();

    uint32_t running = 0;  // restart markers found so far (uniform)
    bool bad = false;
    for (uint64_t chunk = s.ecs_off & ~15ull; chunk < s.ecs_end; chunk += 16ull * kIndexThreads) {
        const uint64_t p0 = chunk + 16ull * tid;
        uint32_t rst = 0, ids = 0;  // bit j: byte p0 + j starts an RSTn marker; ids: 3-bit n per such byte, packed
        uint64_t other = ~0ull;
        if (p0 < s.ecs_end) {
            const uint4 v = *reinterpret_cast<const uint4 *>(input + p0);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
            if ((__vcmpeq4(v.x, 0xffffffffu) | __vcmpeq4(v.y, 0xffffffffu) | __vcmpeq4(v.z, 0xffffffffu) | __vcmpeq4(v.w, 0xffffffffu)) != 0u) {
                const uint32_t nxt = input[p0 + 16];  // the byte behind these 16 (inside the buffer: EOI follows ecs_end)
#pragma unroll
                for (int j = 0; j < 16; j++) {
                    const uint32_t c = (w[j >> 2] >> (8 * (j & 3))) & 0xffu;
                    const uint32_t nb = (j < 15) ? ((w[(j + 1) >> 2] >> (8 * ((j + 1) & 3))) & 0xffu) : nxt;
                    const uint64_t q = p0 + (uint64_t)j;
                    if (c == 0xffu && nb != 0u && nb != 0xffu && q >= s.ecs_off && q < s.ecs_end) {
                        if ((nb & 0xf8u) == 0xd0u) {
                            ids |= (nb & 7u) << (3 * __popc(rst));  // at most 8 markers fit 16 bytes
                            rst |= 1u << j;
                        } else if (nb >= 0xc0u && nb < 0xf0u && other == ~0ull) {
                            other = q;  // 0xff 01..bf / f0..fe is no marker to ParseRestartMarker (entropyparser.cpp:191-196)
                        }
                    }
                }
            }
        }
        // the first marker that is not a restart marker ends the segment: restart markers behind it do not count
        if (other != ~0ull) atomicMin(&first_other, (unsigned long long)other);
        __syncthreads();
        const uint64_t fo = first_other;
        if (fo != ~0ull) {
            uint32_t keep = 0, kids = 0, m = rst, i = 0;
            while (m) {
                const int j = __ffs(m) - 1;
                m &= m - 1;
                if (p0 + (uint64_t)j < fo) {
                    kids |= ((ids >> (3 * i)) & 7u) << (3 * __popc(keep));
                    keep |= 1u << j;
                }
                i++;
            }
            rst = keep;
            ids = kids;
        }
        // exclusive prefix sum of the per-thread counts
        const uint32_t cnt = __popc(rst);
        uint32_t inc = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(kFull, inc, d);
            if (lane >= (uint32_t)d) inc += t;
        }
        if (lane == 31) warp_cnt[warp] = inc;
        __syncthreads();
        uint32_t before = running + inc - cnt, total = 0;
#pragma unroll
        for (int wi = 0; wi < kIndexThreads / 32; wi++) {
            const uint32_t c = warp_cnt[wi];
            if (wi < (int)warp) before += c;
            total += c;
        }
        uint32_t m = rst, i = 0;
        while (m) {
            const int j = __ffs(m) - 1;
            m &= m - 1;
            const uint32_t k = before + i;  // this is restart marker number k of the scan
            const uint64_t pos = p0 + (uint64_t)j;
            if (k < nint) end[k] = pos;
            if (k + 1 < nint) {
                off[k + 1] = pos + 2;
                if (((ids >> (3 * i)) & 7u) != (k & 7u)) bad = true;
            }
            i++;
        }
        running += total;
        __syncthreads();  // warp_cnt is reused by the next step
        if (fo != ~0ull) break;
    }
    const uint64_t seg_end = (first_other != ~0ull) ? (uint64_t)first_other : s.ecs_end;
    if (!__syncthreads_or(bad ? 1 : 0)) {
        if (tid == 0) off[0] = s.ecs_off;
        for (uint32_t k = tid; k < nint; k += kIndexThreads) {
            if (k >= running) end[k] = seg_end;
            if (k > running) off[k] = ~0ull;
        }
    } else {
        // Restart markers out of sequence (damaged stream): the reference resynchronises (entropyparser.cpp:137-199), and what
        // it does is a function of the marker sequence alone -- the bit reader never passes a marker, so after interval k-1
        // the parser stands at, or scans forward to, the first marker behind that interval's data: the expected RSTn is
        // consumed; one that is 4..7 ids behind is dropped with the data after it; one that is 1..3 ids ahead costs
        // interval k (cleared) and stays; the marker that ends the segment costs every interval that is left. Rare and
        // inherently sequential: one thread walks the marker list the parallel pass left in end[] (copied to cln[]).
        const uint32_t nm = running < nint ? running : nint;
        for (uint32_t k = tid; k < nm; k += kIndexThreads) cln[k] = end[k];
        __syncthreads();
        if (tid == 0) {
            uint32_t p = 0, next = 0;
            bool overflow = false;
            off[0] = s.ecs_off;
            end[0] = nm ? cln[0] : seg_end;
            for (uint32_t k = 1; k < nint; k++) {
                bool valid = false;
                for (;;) {
                    if (p >= nm) {  // the end of the segment -- or of the list, if the stream holds more markers than intervals
                        overflow = overflow || running > nint;
                        break;
                    }
                    const uint32_t id = input[cln[p] + 1] & 7u;
                    if (id == next) {
                        off[k] = cln[p] + 2;
                        p++;
                        valid = true;
                        break;
                    }
                    if (((id - next) & 7u) >= 4u) {
                        p++;
                        continue;
                    }
                    break;
                }
                next = (next + 1u) & 7u;
                if (valid) {
                    end[k] = p < nm ? cln[p] : seg_end;
                } else {
                    off[k] = ~0ull;
                    end[k] = seg_end;
                }
            }
            if (overflow) atomicMax(index_status + s.frame, kErrMalformed);  // not resolvable with the list kept here
        }
    }
    __syncthreads();
    for (uint32_t k = tid; k < nint; k += kIndexThreads) {
        const uint64_t o = off[k];
        cln[k] = (o == ~0ull) ? s.clean_base : ((s.clean_base + (o - s.ecs_off) + (uint64_t)kCleanSlackPerInterval * k + 15ull) & ~15ull);
    }
}

}  // namespace

int launch_restart_index(const IndexScan *scans_dev, uint32_t n_scans, uint8_t *input_dev, uint32_t *index_status, void *stream) {
    if (n_scans == 0) return 0;
    restart_index_kernel<<<n_scans, kIndexThreads, 0, (cudaStream_t)stream>>>(scans_dev, input_dev, index_status);
    return (int)cudaGetLastError();
}

int launch_unstuff(const EntropyLaunch &l, void *stream) {
    const uint64_t total = (uint64_t)l.p.n_scans * l.p.intervals_per_scan;
    if (total == 0) return 0;
    if (l.p.indexed) {  // restart-less scans: the interval is the whole entropy coded segment of a frame
        unstuff_long_kernel<<<(uint32_t)total, kLongThreads, 0, (cudaStream_t)stream>>>((uint32_t)total, l.bytes, l.interval_off, l.interval_end,
                                                                                           l.clean_off, l.clean, l.interval_len);
        return (int)cudaGetLastError();
    }
    const uint32_t grid = (uint32_t)((total + kUnstuffWarps - 1) / kUnstuffWarps);
    unstuff_kernel<<<grid, kUnstuffWarps * 32, 0, (cudaStream_t)stream>>>((uint32_t)total, l.bytes, l.interval_off, l.interval_end, l.clean_off,
                                                                           l.clean, l.interval_len);
    return (int)cudaGetLastError();
}

template <bool kIndexed>
static int launch_entropy_impl(const EntropyLaunch &l, void *stream) {
    const uint64_t total = (uint64_t)l.p.n_scans * (kIndexed ? l.p.segs_per_scan : l.p.intervals_per_scan);
    if (total == 0) return 0;
    int dev = 0, sm_count = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
        return (int)cudaGetLastError();
    const uint64_t groups = (total + 31) / 32;
    const uint32_t grid = (uint32_t)(groups < (uint64_t)sm_count ? groups : (uint64_t)sm_count);
    const size_t base_smem = (size_t)kThreads * kStageStride + (size_t)kThreads * 64 + kQzBytes + (kIndexed ? kBdescBytes : 0);
    const size_t lut_bytes = (size_t)l.p.lut_words * 4;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e;
    if (base_smem + lut_bytes <= 227 * 1024) {
        const size_t smem = base_smem + lut_bytes;
        if (smem > 48 * 1024) {
            e = cudaFuncSetAttribute(entropy_decode_kernel<true, kIndexed>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return (int)e;
        }
        entropy_decode_kernel<true, kIndexed><<<grid, kThreads, smem, s>>>(l.p, l.clean, l.clean_off, l.interval_len, l.scans, l.tables, l.coef,
                                                                            l.frame_status, l.overrun_list, l.spec_segments);
    } else {
        // decoder tables too large for shared memory: read from global memory; the staging blocks and the ring alone are
        // beyond the 48 KB a launch gets without opting in
        e = cudaFuncSetAttribute(entropy_decode_kernel<false, kIndexed>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)base_smem);
        if (e != cudaSuccess) return (int)e;
        entropy_decode_kernel<false, kIndexed><<<grid, kThreads, base_smem, s>>>(l.p, l.clean, l.clean_off, l.interval_len, l.scans, l.tables, l.coef,
                                                                                 l.frame_status, l.overrun_list, l.spec_segments);
    }
    e = cudaGetLastError();
    return (int)e;
}

int launch_entropy(const EntropyLaunch &l, void *stream) {
    return l.p.indexed ? launch_entropy_impl<true>(l, stream) : launch_entropy_impl<false>(l, stream);
}

int launch_overrun_verdict(const EntropyLaunch &l, void *stream) {
    const uint64_t total = (uint64_t)l.p.n_scans * l.p.intervals_per_scan;
    if (total == 0) return 0;
    overrun_verdict_kernel<<<8, 128, 0, (cudaStream_t)stream>>>(l.p, l.clean, l.clean_off, l.interval_len, l.scans, l.tables, l.overrun_list,
                                                               l.frame_status);
    return (int)cudaGetLastError();
}

}  // namespace b200jpg
