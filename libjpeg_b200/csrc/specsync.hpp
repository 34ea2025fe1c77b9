// specsync.hpp -- restart-less sequential scans: finding synchronisation points in a Huffman stream that nobody partitioned.
//
// A scan without restart markers is ONE bit stream (EntropyParser never resets anything, codestream/entropyparser.cpp:117-136
// only acts when DRI is set), so the decoder of SequentialScan::ParseMCU / DecodeBlock (codestream/sequentialscan.cpp:381-428,
// 678-773) is a chain over the whole frame. The chain is broken up the way self-synchronising codes allow: the unstuffed
// stream is cut into subsequences of kSpecSeqBits bits; subsequence i is decoded -- lengths only -- from a GUESSED state (a
// block starts exactly at its first bit) up to the first block boundary behind its end, and then again from wherever its
// predecessor really ended, round after round, until no subsequence's exit changes any more. A Huffman decoder that starts in
// the wrong place falls into step with the right one after a few symbols with overwhelming probability, so this takes two
// or three rounds instead of one per subsequence (which is the guaranteed worst case: subsequence 0 starts right). What
// comes out -- for every subsequence the bit where its first block starts, that block's position in the MCU, how many blocks
// it holds and the sum of their DC differences per component -- turns, after prefix sums, into independent work items for
// the output pass: the same decoder as for restart intervals, one item per lane.
//
// The per-subsequence decoder is __host__ __device__ so that the host tests can replay the rounds sequentially and compare
// them with a plain front-to-back walk (tests only; the product path runs it on the device).
#pragma once
#include <cstdint>
#include <vector>

#include "internal.hpp"

#if defined(__CUDACC__)
#define B200JPG_HD __host__ __device__ __forceinline__
#else
#define B200JPG_HD inline
#endif

namespace b200jpg {

#ifndef B200JPG_SPEC_SEQ_BITS
#define B200JPG_SPEC_SEQ_BITS 8192
#endif
constexpr uint32_t kSpecSeqBits = B200JPG_SPEC_SEQ_BITS;  // bits per subsequence (256 words; measured: 4096 -> 8192 bits takes 15 % off the batch AND off a single 4K frame, 16384 nothing more)
constexpr int kSpecMaxBlocksPerMcu = 10;
#ifndef B200JPG_SPEC_RUNUP_BITS
#define B200JPG_SPEC_RUNUP_BITS 2048
#endif
constexpr uint32_t kSpecRunUpBits = B200JPG_SPEC_RUNUP_BITS;   // the first round starts this far in front of a subsequence (see spec_decode)
constexpr size_t kSpecMinBytes = 4096;    // shorter restart-less scans stay one work item (eight subsequences are not worth the rounds)

struct SpecScan {               // what the length-only decoder needs to know about the scan
    const uint32_t *lut;        // two-level tables of the scan's table set (internal.hpp), word offsets below
    uint32_t dc_tab[4], ac_tab[4];   // word offset of the DC / AC table of scan component c
    uint32_t blocks_per_mcu;
    uint32_t blk_period;        // SpecState::blk counts modulo this (spec_table_period, or blocks_per_mcu for the exact position)
    uint8_t comp_of_block[kSpecMaxBlocksPerMcu];  // scan component of block b of an MCU (sequentialscan.cpp:387-424 order)
};

// The smallest p (a divisor of blocks_per_mcu) for which block b and block b + p of the MCU decode with the same DC and AC
// tables. Decoding a stream determines a block's position in the MCU only modulo p: two paths that start on the same bit
// with positions that differ by a multiple of p walk the same bits forever. So the rounds compare and log states with blk
// counted modulo p -- 1 when every component uses the same tables (the reference encoder without colour transformation),
// blocks_per_mcu when the tables tell every position apart -- and the DC differences, which do depend on the exact
// position, are summed by a second walk from the true first block once the entries are known (spec_sync_kernel).
B200JPG_HD uint32_t spec_table_period(const SpecScan &sc) {
    const uint32_t bpm = sc.blocks_per_mcu;
    for (uint32_t p = 1; p < bpm; p++) {
        if (bpm % p) continue;
        bool same = true;
        for (uint32_t b = p; b < bpm && same; b++) {
            const uint32_t c = sc.comp_of_block[b], d = sc.comp_of_block[b - p];
            same = sc.dc_tab[c] == sc.dc_tab[d] && sc.ac_tab[c] == sc.ac_tab[d];
        }
        if (same) return p;
    }
    return bpm;
}

struct SpecState {  // a block boundary on some decoding path
    uint32_t bit;   // position in the unstuffed stream
    uint32_t blk;   // index of the block that starts there inside its MCU
};

struct SpecResult {
    SpecState exit;     // first block boundary at or behind the limit
    uint32_t n_blocks;  // blocks started (and finished) on the way
    int32_t dc_sum[4];  // sum of the DC differences of those blocks, per scan component
};

B200JPG_HD uint32_t spec_word(const uint32_t *w, uint32_t nwords, uint32_t i) { return i < nwords ? w[i] : 0u; }

// the 32 bits at `bit` of a stream of big-endian words (zero bits behind its end, io/bitstream.cpp:96-105)
B200JPG_HD uint32_t spec_window(const uint32_t *w, uint32_t nwords, uint32_t bit) {
    const uint32_t i = bit >> 5, s = bit & 31u;
    const uint32_t a = spec_word(w, nwords, i);
    if (s == 0) return a;
    return (a << s) | (spec_word(w, nwords, i + 1) >> (32u - s));
}

B200JPG_HD uint32_t spec_lookup(const uint32_t *tab, uint32_t hi) {
    uint32_t e = tab[hi >> (32 - kLutL1Bits)];
    if ((e & (31u << 5)) == 0) e = tab[(1u << kLutL1Bits) + ((e >> 10) << (16 - kLutL1Bits)) + ((hi >> 16) & ((1u << (16 - kLutL1Bits)) - 1u))];
    return e;
}

// value bits of entry e in window hi (sequentialscan.cpp:692-696): used for the DC differences only
B200JPG_HD int32_t spec_value(uint32_t e, uint32_t hi) {
    const uint32_t s = e & 31u, len = (e >> 5) & 31u;
    if (s == 0) return 0;
    const uint32_t v = (hi << len) >> (32u - s);
    return (v < (1u << (s - 1))) ? (int32_t)v - (int32_t)((1u << s) - 1u) : (int32_t)v;
}

// Where a subsequence's decoding path stood at the first block boundary behind each of kSpecMarks evenly spaced marks, and
// what was still in front of it there (blocks, DC differences up to the exit). A later round that starts from a corrected
// entry state walks until it stands on one of these states -- the paths have merged -- and takes the rest from the log
// instead of decoding it again: the suffix quantities do not depend on how the path got there.
constexpr int kSpecMarks = 7;
constexpr uint32_t kSpecMarkBits = kSpecSeqBits / (kSpecMarks + 1);
struct SpecLog {
    unsigned long long state[kSpecMarks];  // bit | blk << 32; ~0: not reached
    uint32_t n_after[kSpecMarks];
    int32_t dc_after[kSpecMarks][4];
};

// Decodes whole blocks from `from` until a block boundary at or behind `limit_bit` (or behind the end of the data).
// ONE flat loop, one symbol per iteration (the DC symbol of a block when k == 0, else an AC symbol): the threads of a warp
// run the same few instructions whatever their blocks look like, and only diverge where they finish.
// Block positions advance modulo sc.blk_period: with a period below blocks_per_mcu the states are canonical (blk < period)
// and the DC sums are attributed to the components of those canonical positions, i.e. meaningless; only the block counts
// and the states are used then.
// With a log: `log` holds the marks of this subsequence's previous path (states ~0 before the first round) and receives
// those of the new one; `merged_at` receives the old mark the walk ended on (the exit of the previous round stands and the
// returned counts already include the logged rest), or -1.
// With a run-up (count_from > from.bit): the walk starts somewhere IN FRONT of the subsequence, on a guess; blocks that start in
// front of `count_from` are decoded but not counted, and `*entered` receives the first block boundary at or behind count_from
// -- the subsequence's entry state as this path sees it. A path that has fallen into step during the run-up reports the true
// entry, and its counts and its exit are the true ones without a second walk.
B200JPG_HD SpecResult spec_decode(const SpecScan &sc, const uint32_t *w, uint32_t nwords, uint32_t total_bits, SpecState from, uint32_t limit_bit,
                                  SpecLog *log = nullptr, uint32_t first_mark_bit = 0, int *merged_at = nullptr, uint32_t count_from = 0,
                                  SpecState *entered = nullptr) {
    uint32_t comp_bits = 0;  // two bits per block of an MCU: no indexed local array in the loop
    for (uint32_t b = 0; b < sc.blocks_per_mcu; b++) comp_bits |= (uint32_t)sc.comp_of_block[b] << (2u * b);
    const uint32_t wrap = sc.blk_period;
    // everything the loop needs from the scan description in registers (the struct itself may sit in local memory)
    const uint32_t *const lut = sc.lut;
    const uint32_t dc0 = sc.dc_tab[0], dc1 = sc.dc_tab[1], dc2 = sc.dc_tab[2], dc3 = sc.dc_tab[3];
    const uint32_t ac0 = sc.ac_tab[0], ac1 = sc.ac_tab[1], ac2 = sc.ac_tab[2], ac3 = sc.ac_tab[3];
    uint32_t bit = from.bit, blk = from.blk, k = 0, n = 0;
    // the stream words around `bit` in registers: a symbol has fewer than 32 bits, so at most one new word per step
    // (x2 is a prefetch: the load of a new word has two words' worth of symbols to arrive before the window needs it)
    uint32_t wi = bit >> 5, x0 = spec_word(w, nwords, wi), x1 = spec_word(w, nwords, wi + 1u), x2 = spec_word(w, nwords, wi + 2u);
    // tables of the block the path is in: chosen when the block changes, not per symbol
    uint32_t cur = (comp_bits >> (2u * blk)) & 3u;
    uint32_t dct = cur == 0 ? dc0 : (cur == 1 ? dc1 : (cur == 2 ? dc2 : dc3));
    uint32_t act = cur == 0 ? ac0 : (cur == 1 ? ac1 : (cur == 2 ? ac2 : ac3));
    int32_t s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    int mark = 0, merge_at = -1;   // next mark to pass; the mark the path merged at
    uint32_t next_mark = first_mark_bit;
    if (merged_at) *merged_at = -1;
    if (log) {  // a path that starts behind marks leaves them unreached
        while (mark < kSpecMarks && bit > next_mark) {
            log->state[mark] = ~0ull;
            mark++;
            next_mark += kSpecMarkBits;
        }
    }
    bool counting = entered == nullptr || bit >= count_from;
    if (entered && counting) entered->bit = bit, entered->blk = blk;
    while ((k != 0 || bit < limit_bit) && (k != 0 || bit < total_bits)) {
        if (!counting && k == 0 && bit >= count_from) {  // the run-up is over: this boundary is the entry, counting starts here
            counting = true;
            entered->bit = bit, entered->blk = blk;
            n = 0, s0 = s1 = s2 = s3 = 0;
        }
        if (log && k == 0 && counting && mark < kSpecMarks && bit >= next_mark) {  // at a block boundary: marks passed since the last one
            const unsigned long long here = (unsigned long long)bit | ((unsigned long long)blk << 32);
            while (mark < kSpecMarks && bit >= next_mark && merge_at < 0) {
                if (log->state[mark] == here) {
                    merge_at = mark;
                } else {
                    log->state[mark] = here;
                    log->n_after[mark] = n;  // cumulative for now: turned into "still in front" below
                    log->dc_after[mark][0] = s0, log->dc_after[mark][1] = s1, log->dc_after[mark][2] = s2, log->dc_after[mark][3] = s3;
                    mark++;
                    next_mark += kSpecMarkBits;
                }
            }
            if (merge_at >= 0) break;
        }
        const uint32_t c = cur;
#if defined(__CUDA_ARCH__)
        const uint32_t hi = __funnelshift_l(x1, x0, bit);
#else
        const uint32_t hi = (bit & 31u) ? ((x0 << (bit & 31u)) | (x1 >> (32u - (bit & 31u)))) : x0;
#endif
        const uint32_t e = spec_lookup(lut + (k == 0 ? dct : act), hi);
        if (k == 0) {
            if ((int32_t)e >= 0) {
                const int32_t v = spec_value(e, hi);
                s0 += c == 0 ? v : 0, s1 += c == 1 ? v : 0, s2 += c == 2 ? v : 0, s3 += c == 3 ? v : 0;
                bit += e >> 26;
                k = 1;
            } else {  // an entry that must not be decoded ends the block here: any rule does for a path that is wrong anyway
                bit += 1;
                k = 64;
            }
        } else {
            bit += (e >> 26) & 31u;
            k += (e >> 19) & 127u;  // run + 1, 16 for ZRL, kQzBlockEnds for EOB and error entries
        }
        if (k > 63) {
            k = 0;
            n++;
            blk = blk + 1 == wrap ? 0 : blk + 1;
            cur = (comp_bits >> (2u * blk)) & 3u;
            dct = cur == 0 ? dc0 : (cur == 1 ? dc1 : (cur == 2 ? dc2 : dc3));
            act = cur == 0 ? ac0 : (cur == 1 ? ac1 : (cur == 2 ? ac2 : ac3));
        }
        if ((bit >> 5) != wi) {  // the window moves up by one word
            wi = bit >> 5;
            x0 = x1;
            x1 = x2;
            x2 = spec_word(w, nwords, wi + 2u);
        }
    }
    if (!counting) {  // the walk ended inside the run-up (end of the data): nothing of the subsequence is there
        entered->bit = bit, entered->blk = blk;
        n = 0, s0 = s1 = s2 = s3 = 0;
    }
    if (log) {
        if (merge_at >= 0) {  // the rest of the way is the logged one
            n += log->n_after[merge_at];
            s0 += log->dc_after[merge_at][0], s1 += log->dc_after[merge_at][1], s2 += log->dc_after[merge_at][2], s3 += log->dc_after[merge_at][3];
            if (merged_at) *merged_at = merge_at;
        } else {  // marks behind the exit were not reached on this path
            for (int m = mark; m < kSpecMarks; m++) log->state[m] = ~0ull;
        }
        for (int m = 0; m < mark && m < (merge_at >= 0 ? merge_at : kSpecMarks); m++) {  // cumulative -> what was still in front
            log->n_after[m] = n - log->n_after[m];
            log->dc_after[m][0] = s0 - log->dc_after[m][0], log->dc_after[m][1] = s1 - log->dc_after[m][1];
            log->dc_after[m][2] = s2 - log->dc_after[m][2], log->dc_after[m][3] = s3 - log->dc_after[m][3];
        }
    }
    SpecResult r;
    r.exit.bit = bit, r.exit.blk = blk;
    r.n_blocks = n;
    r.dc_sum[0] = s0, r.dc_sum[1] = s1, r.dc_sum[2] = s2, r.dc_sum[3] = s3;
    return r;
}

static_assert(sizeof(SpecLog) % 8 == 0, "SpecLog arrays keep their 64-bit members aligned");

// One work item of the output pass: blocks [first_block, first_block + n_blocks) of the scan start at bit `bit`
struct SpecSegment {
    uint32_t bit;
    uint32_t first_block;
    uint32_t n_blocks;
    int32_t pred[4];  // DC predictors of the scan components in front of the first block
    uint32_t pad;
};

static_assert(sizeof(SpecSegment) == 32, "two 16-byte loads per work item (entropy_decode_kernel)");

// Host replay of spec_sync_kernel's rounds for one scan (tests only; specsync_sm100.cu). Returns the number of rounds.
int spec_sync_host_replay(const SpecScan &sc, const uint32_t *words, uint32_t len_bytes, uint32_t total_mcus, std::vector<SpecSegment> &segs);

}  // namespace b200jpg
