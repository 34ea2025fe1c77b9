// specsync_sm100.cu -- synchronisation points of restart-less sequential scans (see specsync.hpp).
//
// spec_sync_kernel: one CTA per scan. The scan's decoder tables go to shared memory; the threads take the subsequences of
// kSpecSeqBits bits in turns. Round 0 decodes every subsequence from the guess "a block starts at my first bit"; every later
// round re-decodes exactly those whose entry state -- the exit state of their predecessor -- has changed. The exits live in
// one array that is read and written without ordering inside a round (an 8-byte store is atomic; a stale read is caught by
// the `changed` vote, which forces another round), so the iteration is chaotic but monotone: subsequence 0 starts right, a
// right entry gives a right exit, and a Huffman decoder that starts wrong falls into step with the right one after a few
// symbols -- two or three rounds for real images, nseq rounds in the worst case. Then one pass of prefix sums (block counts
// -> first block index, DC differences -> predictors) turns the subsequences into the SpecSegment work items that
// entropy_decode_kernel<.., kIndexed = true> decodes one per lane.
#include <cuda_runtime.h>

#include <cstdint>

#include "internal.hpp"
#include "specsync.hpp"

namespace b200jpg {
namespace {

constexpr int kSyncThreads = 512;
// kMinCtas = CTAs per SM the register allocation aims at: 3 (40 registers, a few spills) wins when many scans are in flight,
// 2 (64 registers) is the shorter way through one scan
template <int kMinCtas>
__global__ void __launch_bounds__(kSyncThreads, kMinCtas)
spec_sync_kernel(ScanClassParams p, const uint8_t *__restrict__ clean, const uint64_t *__restrict__ clean_off,
                 const uint32_t *__restrict__ interval_len, const uint8_t *__restrict__ tables, SpecSegment *__restrict__ segs,
                 unsigned long long *__restrict__ exits, unsigned long long *__restrict__ entries, uint32_t *__restrict__ counts,
                 int32_t *__restrict__ dc_sums, SpecLog *__restrict__ logs) {
    extern __shared__ uint32_t s_lut[];
    __shared__ int s_changed;
    const uint32_t j = blockIdx.x;  // scan
    const uint32_t tid = threadIdx.x;
    const uint32_t *g_lut = reinterpret_cast<const uint32_t *>(tables + kTableHeaderBytes);
    const uint16_t *lut_off = reinterpret_cast<const uint16_t *>(tables + 16);
    for (uint32_t i = tid; i < p.lut_words; i += kSyncThreads) s_lut[i] = g_lut[i];
    SpecScan sc;
    sc.lut = s_lut;
    sc.blocks_per_mcu = 0;
    for (int c = 0; c < p.ns; c++) {
        sc.dc_tab[c] = lut_off[p.dc_slot[c]];
        sc.ac_tab[c] = lut_off[4 + p.ac_slot[c]];
        for (int b = 0; b < p.mw[c] * p.mh[c]; b++) sc.comp_of_block[sc.blocks_per_mcu++] = (uint8_t)c;
    }
    sc.blk_period = spec_table_period(sc);
    const uint32_t len_bytes = interval_len[j] & kIntervalLenMask;
    const uint32_t total_bits = len_bytes * 8u, nwords = (len_bytes + 3u) / 4u;
    const uint32_t *w = reinterpret_cast<const uint32_t *>(clean + clean_off[j]);
    const uint32_t cap = p.segs_per_scan;
    uint32_t nseq = (total_bits + kSpecSeqBits - 1u) / kSpecSeqBits;
    if (nseq > cap) nseq = cap;  // cannot happen: unstuffing only shrinks the data the host sized the arrays for
    SpecSegment *seg = segs + (size_t)j * cap;
    unsigned long long *ex = exits + (size_t)j * cap, *en = entries + (size_t)j * cap;
    uint32_t *cnt = counts + (size_t)j * cap;
    int32_t *ds = dc_sums + (size_t)j * cap * 4u;
    SpecLog *lg = logs + (size_t)j * cap;
    if (tid == 0) s_changed = 1;
    for (uint32_t i = tid; i < nseq; i += kSyncThreads) {
        ex[i] = ~0ull;
        en[i] = ~0ull;
        for (int m = 0; m < kSpecMarks; m++) lg[i].state[m] = ~0ull;
    }
    __syncthreads();
    for (uint32_t round = 0; s_changed; round++) {
        __syncthreads();
        if (tid == 0) s_changed = 0;
        __syncthreads();
        bool changed = false;
        for (uint32_t i = tid; i < nseq; i += kSyncThreads) {
            unsigned long long entry;
            const bool run_up = round == 0 && i != 0;
            if (i == 0) entry = 0ull;                                         // the scan starts with block 0 of MCU 0 at bit 0
            else if (round == 0) entry = (unsigned long long)(i * kSpecSeqBits - kSpecRunUpBits);  // the guess: a block starts here
            else entry = *reinterpret_cast<volatile unsigned long long *>(ex + i - 1);
            if (!run_up && (entry == en[i] || entry == ~0ull)) continue;
            SpecState from, entered;
            from.bit = (uint32_t)entry;
            from.blk = (uint32_t)(entry >> 32);
            int merged_at;
            const SpecResult r = spec_decode(sc, w, nwords, total_bits, from, (i + 1u) * kSpecSeqBits, lg + i, i * kSpecSeqBits + kSpecMarkBits, &merged_at,
                                             run_up ? i * kSpecSeqBits : 0u, run_up ? &entered : nullptr);
            // the entry this walk really had: after a run-up, the first block boundary inside the subsequence as the walk found it
            en[i] = run_up ? ((unsigned long long)entered.bit | ((unsigned long long)entered.blk << 32)) : entry;
            cnt[i] = r.n_blocks;
            ds[4 * i + 0] = r.dc_sum[0], ds[4 * i + 1] = r.dc_sum[1], ds[4 * i + 2] = r.dc_sum[2], ds[4 * i + 3] = r.dc_sum[3];
            if (merged_at >= 0) continue;  // the path joined the previous round's: its exit stands
            const unsigned long long out = (unsigned long long)r.exit.bit | ((unsigned long long)r.exit.blk << 32);
            if (out != ex[i]) {
                *reinterpret_cast<volatile unsigned long long *>(ex + i) = out;
                changed = true;
            }
        }
        if (changed) s_changed = 1;
        __syncthreads();
    }
    const uint32_t total_blocks = p.total_mcus * sc.blocks_per_mcu;
    if (sc.blk_period != sc.blocks_per_mcu) {
        // the rounds knew block positions modulo the table period only, so their DC sums went to the wrong components.
        // The first block of every subsequence (prefix sums of the counts, into the exits, which are done with) gives its
        // true position; one more walk from there sums the DC differences per component.
        if (tid == 0) {
            uint32_t first = 0;
            for (uint32_t i = 0; i < nseq; i++) {
                ex[i] = first < total_blocks ? first : ~0ull;
                if (first < total_blocks) first += cnt[i] < total_blocks - first ? cnt[i] : total_blocks - first;
            }
        }
        __syncthreads();
        sc.blk_period = sc.blocks_per_mcu;
        for (uint32_t i = tid; i < nseq; i += kSyncThreads) {
            const unsigned long long first = ex[i];
            if (first == ~0ull) continue;
            SpecState from;
            from.bit = (uint32_t)en[i];
            from.blk = (uint32_t)first % sc.blocks_per_mcu;
            const SpecResult r = spec_decode(sc, w, nwords, total_bits, from, (i + 1u) * kSpecSeqBits);
            ds[4 * i + 0] = r.dc_sum[0], ds[4 * i + 1] = r.dc_sum[1], ds[4 * i + 2] = r.dc_sum[2], ds[4 * i + 3] = r.dc_sum[3];
        }
        __syncthreads();
    }
    // prefix sums over the subsequences: first block index and DC predictors. Sequential in one thread: a few thousand
    // additions per scan next to megabits of Huffman decoding.
    if (tid == 0) {
        uint32_t first = 0, last_used = 0;
        int32_t pred[4] = {0, 0, 0, 0};
        for (uint32_t i = 0; i < cap; i++) {
            SpecSegment s;
            s.bit = 0, s.first_block = first, s.n_blocks = 0, s.pad = 0;
            s.pred[0] = pred[0], s.pred[1] = pred[1], s.pred[2] = pred[2], s.pred[3] = pred[3];
            if (i < nseq && first < total_blocks) {
                uint32_t n = cnt[i];
                if (n > total_blocks - first) n = total_blocks - first;  // blocks decoded out of the padding behind the last MCU
                s.bit = (uint32_t)en[i];
                s.n_blocks = n;
                if (n) last_used = i;
                first += n;
                pred[0] += ds[4 * i + 0], pred[1] += ds[4 * i + 1], pred[2] += ds[4 * i + 2], pred[3] += ds[4 * i + 3];
            }
            seg[i] = s;
        }
        // the data ends in front of the last MCU (a cut stream): the reference goes on decoding zero bits (io/bitstream.cpp:
        // 96-105); the last segment takes the blocks that are left and does the same
        if (first < total_blocks) seg[nseq ? last_used : 0].n_blocks += total_blocks - first;
    }
}

}  // namespace

int launch_spec_sync(const EntropyLaunch &l, void *stream) {
    if (l.p.n_scans == 0) return 0;
    const size_t smem = (size_t)l.p.lut_words * 4;
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const bool many = l.p.n_scans >= 2u * (uint32_t)sms;  // more CTAs than two per SM: occupancy counts more than the single path
    auto kernel = many ? spec_sync_kernel<3> : spec_sync_kernel<2>;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    kernel<<<l.p.n_scans, kSyncThreads, smem, (cudaStream_t)stream>>>(l.p, l.clean, l.clean_off, l.interval_len, l.tables, l.spec_segments, l.spec_exits,
                                                                      l.spec_entries, l.spec_counts, l.spec_dc_sums, l.spec_logs);
    return (int)cudaGetLastError();
}

}  // namespace b200jpg
unsigned long long g_spec_replay_bits = 0;
unsigned long long g_spec_replay_merges[b200jpg::kSpecMarks] = {};
namespace b200jpg {  // host replay only: bits walked (a merged walk counts up to the merge), walks that merged at each mark

// Host replay of the same rounds (tests only): fills `segs` for one scan given its unstuffed words; returns the rounds used.
int spec_sync_host_replay(const SpecScan &scan, const uint32_t *w, uint32_t len_bytes, uint32_t total_mcus, std::vector<SpecSegment> &segs) {
    SpecScan sc = scan;
    sc.blk_period = spec_table_period(sc);
    const uint32_t total_bits = len_bytes * 8u, nwords = (len_bytes + 3u) / 4u;
    const uint32_t nseq = (total_bits + kSpecSeqBits - 1u) / kSpecSeqBits;
    std::vector<unsigned long long> ex(nseq, ~0ull), en(nseq, ~0ull);
    std::vector<uint32_t> cnt(nseq, 0);
    std::vector<int32_t> ds(4 * (size_t)nseq, 0);
    std::vector<SpecLog> logs(nseq);
    for (auto &l : logs)
        for (int m = 0; m < kSpecMarks; m++) l.state[m] = ~0ull;
    int rounds = 0;
    for (bool changed = true; changed; rounds++) {
        changed = false;
        const std::vector<unsigned long long> prev = ex;  // a synchronous round: everybody sees last round's exits
        for (uint32_t i = 0; i < nseq; i++) {
            const bool run_up = rounds == 0 && i != 0;
            unsigned long long entry = i == 0 ? 0ull : (rounds == 0 ? (unsigned long long)(i * kSpecSeqBits - kSpecRunUpBits) : prev[i - 1]);
            if (!run_up && (entry == en[i] || entry == ~0ull)) continue;
            SpecState from, entered;
            from.bit = (uint32_t)entry, from.blk = (uint32_t)(entry >> 32);
            int merged_at;
            const SpecResult r = spec_decode(sc, w, nwords, total_bits, from, (i + 1u) * kSpecSeqBits, &logs[i], i * kSpecSeqBits + kSpecMarkBits, &merged_at,
                                             run_up ? i * kSpecSeqBits : 0u, run_up ? &entered : nullptr);
            en[i] = run_up ? ((unsigned long long)entered.bit | ((unsigned long long)entered.blk << 32)) : entry;
            ::g_spec_replay_bits += r.exit.bit > from.bit ? r.exit.bit - from.bit : 0;
            cnt[i] = r.n_blocks;
            for (int c = 0; c < 4; c++) ds[4 * i + c] = r.dc_sum[c];
            if (merged_at >= 0) {
                ::g_spec_replay_merges[merged_at]++;
                continue;
            }
            const unsigned long long out = (unsigned long long)r.exit.bit | ((unsigned long long)r.exit.blk << 32);
            if (out != ex[i]) ex[i] = out, changed = true;
        }
    }
    const uint32_t total_blocks = total_mcus * sc.blocks_per_mcu;
    if (sc.blk_period != sc.blocks_per_mcu) {  // the DC sums again from every subsequence's true first block (spec_sync_kernel)
        uint32_t first = 0;
        SpecScan exact = sc;
        exact.blk_period = sc.blocks_per_mcu;
        for (uint32_t i = 0; i < nseq && first < total_blocks; i++) {
            const SpecState from{(uint32_t)en[i], first % sc.blocks_per_mcu};
            const SpecResult r = spec_decode(exact, w, nwords, total_bits, from, (i + 1u) * kSpecSeqBits);
            ::g_spec_replay_bits += r.exit.bit > from.bit ? r.exit.bit - from.bit : 0;
            for (int c = 0; c < 4; c++) ds[4 * i + c] = r.dc_sum[c];
            first += cnt[i] < total_blocks - first ? cnt[i] : total_blocks - first;
        }
    }
    segs.assign(nseq, SpecSegment{});
    uint32_t first = 0, last_used = 0;
    int32_t pred[4] = {0, 0, 0, 0};
    for (uint32_t i = 0; i < nseq; i++) {
        SpecSegment s{};
        s.first_block = first;
        for (int c = 0; c < 4; c++) s.pred[c] = pred[c];
        if (first < total_blocks) {
            uint32_t n = cnt[i];
            if (n > total_blocks - first) n = total_blocks - first;
            s.bit = (uint32_t)en[i];
            s.n_blocks = n;
            if (n) last_used = i;
            first += n;
            for (int c = 0; c < 4; c++) pred[c] += ds[4 * i + c];
        }
        segs[i] = s;
    }
    if (segs.empty()) segs.assign(1, SpecSegment{});
    if (first < total_blocks) segs[nseq ? last_used : 0].n_blocks += total_blocks - first;
    return rounds;
}

}  // namespace b200jpg
