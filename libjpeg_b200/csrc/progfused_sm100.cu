// progfused_sm100.cu -- progressive (SOF2) frames decoded COMPONENT BY COMPONENT instead of scan by scan.
//
// The scans of a progressive frame build on each other, but only inside one 8x8 block: what a scan does to a block depends on
// what the earlier scans left in THAT block and on nothing else (RefinementScan::DecodeBlock codestream/refinementscan.cpp:
// 584-690 looks at the block's own coefficients; the EOB runs and DC predictors of SequentialScan::DecodeBlock codestream/
// sequentialscan.cpp:678-773 are per scan). Every scan is its own bit stream. So instead of ten launches that each drag the
// whole coefficient store through HBM (one restart interval per lane, read-modify-write in place), a lane here owns a restart
// interval of ONE component and carries one bit reader per scan of that component: block after block it runs the block through
// all of the component's AC scans in file order -- in a 128-byte staging block in shared memory, already dequantised (the scans
// only ever add multiples of 1 << Al, so value x quantiser can be accumulated directly) --, adds the DC value and hands the
// finished block to the same warp-cooperative flush as the sequential kernel. The coefficient store is written exactly once
// and never read; there is no dequantisation pass and no memset.
//   pf_dc_kernel : the interleaved DC scans (first pass + refinements, sequentialscan.cpp:682-701, refinementscan.cpp:588-592)
//                  -> one int16 level per block in a dense side plane (1/64 of the coefficient store); blocks of the MCU-padded
//                  grid that no AC scan covers are completed here (DC + zeros).
//   pf_ac_kernel : per component, all its AC scans (first passes with EOB runs :704-772, refinements with correction bits
//                  refinementscan.cpp:594-690).
// The host uses this path when the frame's scan script has that shape -- every scan either an interleaved DC scan of all
// components or a single-component AC scan, restart intervals equal within each group (the reference encoder's `-v` script, and
// the usual ones) -- and the scan-by-scan kernels of progressive_sm100.cu otherwise.
#include <cuda_runtime.h>

#include <cstdint>

#include "internal.hpp"

namespace b200jpg {
namespace {

constexpr int kPfThreads = 256;
constexpr int kStage = 144;  // bytes per lane: 128 + 16 pad -> conflict-free 16-byte accesses (like the sequential kernel)
constexpr uint32_t kErrMalformed = 1038u;

// Bit reader over the unstuffed big-endian words of one interval (L1-cached global loads, one word of lookahead); behind the
// end it hands out zero bits like the reference's reader in front of a marker (io/bitstream.cpp:96-105).
struct Bits {
    const uint32_t *w;
    uint32_t nwords, bp, x0, x1, x2;
    __device__ __forceinline__ uint32_t word(uint32_t i) const { return i < nwords ? __ldg(w + i) : 0u; }
    __device__ __forceinline__ void open(const uint8_t *p, uint32_t len_bytes) { resume(p, (len_bytes + 3u) / 4u, 0u); }
    // picks the stream up again at bit `at` (the AC kernel parks the readers of the scans it is not in in shared memory)
    __device__ __forceinline__ void resume(const uint8_t *p, uint32_t words, uint32_t at) {
        w = reinterpret_cast<const uint32_t *>(p);
        nwords = words;
        bp = at;
        const uint32_t wi = at >> 5;
        x0 = word(wi), x1 = word(wi + 1u), x2 = word(wi + 2u);
    }
    __device__ __forceinline__ uint32_t window() const { return __funnelshift_l(x1, x0, bp); }
    __device__ __forceinline__ void skip(uint32_t n) {  // n < 32
        const uint32_t was = bp >> 5;
        bp += n;
        const uint32_t wi = bp >> 5;
        if (wi != was) x0 = x1, x1 = x2, x2 = word(wi + 2u);
    }
    __device__ __forceinline__ uint32_t get(uint32_t n) {  // n <= 24
        const uint32_t v = n ? (window() >> (32u - n)) : 0u;
        skip(n);
        return v;
    }
};

__device__ __forceinline__ uint32_t lut_entry(const uint32_t *lut, uint32_t hi) {
    uint32_t e = lut[hi >> (32 - kLutL1Bits)];
    if ((e & (31u << 5)) == 0) e = lut[(1u << kLutL1Bits) + ((e >> 10) << (16 - kLutL1Bits)) + ((hi >> 16) & ((1u << (16 - kLutL1Bits)) - 1u))];
    return e;
}
__device__ __forceinline__ int extend(uint32_t v, uint32_t s) {  // sequentialscan.cpp:692-696 / 757-762
    return (v < (1u << (s - 1))) ? (int)v + (int)((~0u) << s) + 1 : (int)v;
}

__device__ __forceinline__ void sts_zero16(uint32_t a) { asm volatile("st.shared.v4.u32 [%0], {%1,%1,%1,%1};" ::"r"(a), "r"(0u) : "memory"); }
__device__ __forceinline__ uint4 lds16(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_h(uint32_t a, int v) { asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "h"((short)v) : "memory"); }
__device__ __forceinline__ int lds_h(uint32_t a) {
    int v;
    asm volatile("ld.shared.s16 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_q(uint32_t a, uint64_t v) { asm volatile("st.shared.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }
__device__ __forceinline__ uint64_t lds_q(uint32_t a) {
    uint64_t v;
    asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(a) : "memory");
    return v;
}

// =====================================================================================================
// DC scans: one restart interval of the interleaved DC scans per lane
// =====================================================================================================
__global__ void __launch_bounds__(kPfThreads)
pf_dc_kernel(PfLaunch L) {
    extern __shared__ uint32_t s_lut[];  // tables of the first DC scan (the refinements read raw bits)
    const PfScan &first = L.scan[0];
    const uint32_t *g_lut = reinterpret_cast<const uint32_t *>(first.tables + kTableHeaderBytes);
    for (uint32_t i = threadIdx.x; i < first.lut_words; i += kPfThreads) s_lut[i] = g_lut[i];
    __syncthreads();
    const uint16_t *lut_off = reinterpret_cast<const uint16_t *>(first.tables + 16);
    const uint64_t g = (uint64_t)blockIdx.x * kPfThreads + threadIdx.x;
    if (g >= (uint64_t)L.n_frames * L.intervals) return;
    const uint32_t j = (uint32_t)(g / L.intervals), iv = (uint32_t)(g % L.intervals);
    const ClassScan &cs = L.frames[j];
    Bits b[kPfMaxScans];
    bool present[kPfMaxScans];
#pragma unroll
    for (int s = 0; s < kPfMaxScans; s++) {
        present[s] = false;
        if (s < L.n_scans) {
            const uint32_t raw = L.scan[s].interval_len[g];
            present[s] = !(raw & kIntervalLenAbsent);
            b[s].open(L.clean + L.scan[s].clean_off[g], raw & kIntervalLenMask);
        }
    }
    const uint32_t mcu0 = iv * L.dri;
    const uint32_t nmcu = (L.total_mcus - mcu0 < L.dri) ? (L.total_mcus - mcu0) : L.dri;
    uint32_t mx = mcu0 % L.mcu_cols, my = mcu0 / L.mcu_cols;
    int pred[4] = {0, 0, 0, 0};
    bool bad = false;
    for (uint32_t mi = 0; mi < nmcu; mi++) {
#pragma unroll
        for (int c = 0; c < 4; c++) {
            if (c >= L.ns) break;
            const uint32_t *dc = s_lut + lut_off[first.dc_slot[c]];
            for (int y = 0; y < L.mh[c]; y++)
                for (int x = 0; x < L.mw[c]; x++) {
                    int level = 0;
                    if (present[0] && !bad) {  // first pass: sequentialscan.cpp:682-701
                        const uint32_t e = lut_entry(dc, b[0].window());
                        if ((int)e < 0) {
                            bad = true;
                        } else {
                            b[0].skip((e >> 5) & 31u);
                            const uint32_t sz = e & 31u;
                            if (sz) pred[c] += extend(b[0].get(sz), sz);
                        }
                        const long long lv = (long long)pred[c] * (1ll << first.al);
                        if (lv < -32768 || lv > 32767) bad = true;  // beyond the int16 side plane (DESIGN.md section 7)
                        level = (int)lv;
                    }
#pragma unroll
                    for (int s = 1; s < kPfMaxScans; s++)  // refinements: one raw bit per block, refinementscan.cpp:588-592
                        if (s < L.n_scans && present[s]) level |= (int)(b[s].get(1) << L.scan[s].al);
                    if (level < -32768 || level > 32767) bad = true;
                    const uint32_t bx = mx * L.mw[c] + x, by = my * L.mh[c] + y;
                    const uint64_t blk = cs.coef_base[c] / 64u + (uint64_t)by * L.bw[c] + bx;
                    L.dcplane[blk] = (int16_t)level;
                    if (bx >= L.ac_cols[c] || by >= L.ac_rows[c]) {
                        // a block of the MCU-padded grid that the component's own (non-interleaved) scans never visit:
                        // complete it here -- the dequantised DC and 63 zeros
                        const int v = level * (int)L.dc_quant[c];
                        if (v > 32767 || v < -32768) bad = true;
                        uint4 *d = reinterpret_cast<uint4 *>(L.coef + cs.coef_base[c] + ((uint64_t)by * L.bw[c] + bx) * 64u);
                        d[0] = make_uint4((uint32_t)v & 0xffffu, 0u, 0u, 0u);
#pragma unroll
                        for (int i = 1; i < 8; i++) d[i] = make_uint4(0u, 0u, 0u, 0u);
                    }
                }
        }
        if (++mx == L.mcu_cols) mx = 0, my++;
    }
    if (bad) atomicMax(L.frame_status + cs.frame, kErrMalformed);
}

// =====================================================================================================
// AC scans of one component: one restart interval (of that component's block grid) per lane
// =====================================================================================================
// shared memory: [staging: kPfThreads * kStage][parked readers: n_scans * 3 * kPfThreads words][meta: 2 words per scan]
//                [per scan: qz pairs (128 words)][one LUT per DISTINCT AC table (PfScan::lut_share)]
// Registers are what limits the warps per SM here, and a lane is inside ONE scan at a time: the bit readers of the other
// scans are parked in shared memory as (first word, words, bit position) and re-opened -- three L2 loads -- when the walk
// over the scans of a block comes to them.
__global__ void __launch_bounds__(kPfThreads, 3)
pf_ac_kernel(PfLaunch L) {
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t s_base = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t s_stage = s_base + threadIdx.x * kStage;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t s_flush_sub = (lane & 7u) << 4;
    const uint32_t s_flush = s_base + ((threadIdx.x & ~31u) + (lane >> 3)) * kStage + s_flush_sub;
    uint32_t *s_park = reinterpret_cast<uint32_t *>(smem + kPfThreads * kStage) + threadIdx.x;  // [scan][4][thread]: first word, words, bit position, blocks left of an EOB run
    uint32_t *s_meta = reinterpret_cast<uint32_t *>(smem + kPfThreads * kStage) + (uint32_t)L.n_scans * 4u * kPfThreads;
    // per scan: the (q, byte offset) pairs of the component's quantiser (already << Al, parse.cpp build_table_set) and the AC table
    uint32_t *s_tab = s_meta + 2 * kPfMaxScans;
    {
        uint32_t at = 0;
        uint32_t lut_of[kPfMaxScans];
#pragma unroll
        for (int s = 0; s < kPfMaxScans; s++) {
            lut_of[s] = 0;
            if (s < L.n_scans) {
                const PfScan &sc = L.scan[s];
                const uint32_t *g_qz = reinterpret_cast<const uint32_t *>(sc.tables + 32) + (uint32_t)(kQzEntries * 2) * sc.q_slot;
                const uint32_t *g_lut = reinterpret_cast<const uint32_t *>(sc.tables + kTableHeaderBytes);
                const uint16_t *lut_off = reinterpret_cast<const uint16_t *>(sc.tables + 16);
                for (uint32_t i = threadIdx.x; i < 128u; i += kPfThreads) s_tab[at + i] = g_qz[i];  // the pairs of k = 0..63
                if (threadIdx.x == 0) s_meta[2 * s] = at;
                at += 128u;
                if (sc.lut_share == s) {  // the first scan with this table holds the copy
                    lut_of[s] = at;
                    for (uint32_t i = threadIdx.x; i < sc.lut_words; i += kPfThreads) s_tab[at + i] = g_lut[i];
                    at += sc.lut_words;
                } else {
#pragma unroll
                    for (int t = 0; t < kPfMaxScans; t++)
                        if (t == sc.lut_share) lut_of[s] = lut_of[t];
                }
                if (threadIdx.x == 0) s_meta[2 * s + 1] = lut_of[s] + lut_off[4 + sc.ac_slot];
            }
        }
#pragma unroll
        for (int i = 0; i < 9; i++) sts_zero16(s_stage + 16 * i);
    }
    const uint64_t total = (uint64_t)L.n_frames * L.intervals;
    const uint64_t g = (uint64_t)blockIdx.x * kPfThreads + threadIdx.x;
    const bool lane_valid = g < total;
    const uint64_t gg = lane_valid ? g : 0;
    const uint32_t j = (uint32_t)(gg / L.intervals), iv = (uint32_t)(gg % L.intervals);
    const ClassScan &cs = L.frames[j];
    uint32_t present = 0;  // bit s: this lane's interval of scan s is in the stream
#pragma unroll
    for (int s = 0; s < kPfMaxScans; s++) {
        if (s < L.n_scans) {
            const uint32_t raw = lane_valid ? L.scan[s].interval_len[gg] : kIntervalLenAbsent;
            const bool there = !(raw & kIntervalLenAbsent);
            present |= there ? (1u << s) : 0u;
            s_park[(4 * s + 0) * kPfThreads] = (uint32_t)(L.scan[s].clean_off[gg] >> 2);  // first word (16-byte aligned offsets)
            s_park[(4 * s + 1) * kPfThreads] = there ? ((raw & kIntervalLenMask) + 3u) / 4u : 0u;
            s_park[(4 * s + 2) * kPfThreads] = 0u;
            s_park[(4 * s + 3) * kPfThreads] = 0u;
        }
    }
    __syncthreads();
    const uint32_t mcu0 = iv * L.dri;
    uint32_t nblk = 0;
    if (lane_valid) nblk = (L.total_mcus - mcu0 < L.dri) ? (L.total_mcus - mcu0) : L.dri;
    uint32_t bx = mcu0 % L.mcu_cols, by = mcu0 / L.mcu_cols;
    const uint64_t plane = cs.coef_base[0];
    const int dcq = (int)L.dc_quant[0];
    uint32_t ovf = 0;   // | (v + 32768): bits 16.. set when a dequantised coefficient left the int16 range
    bool bad = false;

    for (uint32_t bi = 0; bi < L.dri; bi++) {
        const bool has = bi < nblk;
        unsigned long long H = 0ull;  // bit k: coefficient k (zig-zag) of this block is non-zero so far
        // The scans of the script are the same for every lane, so the walk over them is uniform; inside a scan every lane is
        // somewhere else in ITS block, so the symbol loops are voted: one Huffman symbol per warp-convergent iteration (like the
        // sequential kernel), lanes that are through wait for the others in the vote, not in divergent code.
#pragma unroll
        for (int s = 0; s < kPfMaxScans; s++) {
            if (s >= L.n_scans) break;
            const PfScan &sc = L.scan[s];
            const uint32_t *lut = s_tab + s_meta[2 * s + 1];
            const uint32_t qz = (uint32_t)__cvta_generic_to_shared(s_tab + s_meta[2 * s]);  // shared-space address of the pairs
            const int ss = sc.ss, se = sc.se;
            // an interval the stream does not contain leaves the block as the other scans make it
            bool active = has && !bad && ((present >> s) & 1u);
            // the lane reads bits of this scan in this block unless it sits in an EOB run of a first pass
            uint32_t run_left = s_park[(4 * s + 3) * kPfThreads];  // blocks of an EOB run still to come (this one included)
            const uint32_t run_was = run_left;
            const bool reads = active && !(sc.ah == 0 && run_left > 0);
            Bits r;
            r.resume(L.clean, 0u, 0u);
            if (reads) r.resume(L.clean + 4ull * s_park[(4 * s + 0) * kPfThreads], s_park[(4 * s + 1) * kPfThreads], s_park[(4 * s + 2) * kPfThreads]);
            int k = ss;
            if (sc.ah == 0) {
                // ---- first pass of the band: sequentialscan.cpp:704-772
                if (active && run_left > 0) {
                    run_left--;
                    active = false;
                }
                while (__any_sync(0xffffffffu, active)) {
                    if (active) {
                        // one symbol, in one straight line whatever its kind (coefficient, ZRL, EOBn): the lanes of a warp stay
                        // together inside the iteration
                        const uint32_t e = lut_entry(lut, r.window());
                        r.skip((e >> 5) & 31u);
                        const uint32_t run = (e >> 10) & 15u, sz = e & 31u;
                        const bool eob = sz == 0 && run != 15;
                        const uint32_t bits = r.get(sz ? sz : (eob ? run : 0u));  // value bits, or the length of an EOB run
                        const int kk = k + (int)run;                             // ZRL: 15 zeros and the (zero) "coefficient" behind them
                        if ((int)e < 0 || (sz != 0 && kk >= 64)) {  // undefined code / the reference tests against 64, not against Se
                            bad = true;
                            active = false;
                        } else {
                            if (sz != 0) {
                                uint2 pq;
                                asm("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(pq.x), "=r"(pq.y) : "r"(qz + 8u * (uint32_t)kk));
                                // |level| < 2^15 and the table caps q << Al at 32769 (build_table_set): no int32 wrap
                                const int d = extend(bits, sz) * (int)pq.x;
                                ovf |= (uint32_t)(d + 32768);
                                sts_h(s_stage + pq.y, d);
                                H |= 1ull << kk;
                            }
                            k = kk + 1;
                            if (eob) run_left = ((1u << run) | bits) - 1u;  // EOBn; this block is part of the run
                            if (eob || k > se) active = false;
                        }
                    }
                }
            } else {
                // ---- refinement of the band: refinementscan.cpp:594-690. The walk over the band is done on the mask of
                // non-zero coefficients instead of coefficient by coefficient: a symbol (run r, size 0 / 1) places its value on
                // the (r+1)-th still-zero position at or behind k; every non-zero position passed on the way takes one
                // correction bit, in order. `pending` collects the positions that still owe a correction bit; they are paid
                // one per voted iteration as well, before the lane decodes its next symbol.
                const unsigned long long band = ((se >= 63) ? ~0ull : ((1ull << (se + 1)) - 1ull)) & ~((1ull << ss) - 1ull);
                unsigned long long pending = 0ull;
                bool tail = active && run_left > 0;  // inside an EOB run: the whole band only takes correction bits
                if (tail) {
                    pending = H & band;
                    active = false;
                }
                while (__any_sync(0xffffffffu, active || pending != 0ull)) {
                    // every iteration: a lane that owes no correction bit decodes its next symbol, and then every lane that owes
                    // one (also the one that has just decoded) pays one -- two straight pieces instead of two diverging ones
                    if (pending == 0ull && active) {
                        // one symbol, straight through for every kind (new coefficient, ZRL, EOBn, a size the reference ignores)
                        const uint32_t e = lut_entry(lut, r.window());
                        r.skip((e >> 5) & 31u);
                        const uint32_t sz = e & 31u;
                        const bool eob = sz == 0 && ((e >> 10) & 15u) != 15u;
                        // the reference warns about sizes other than 0 / 1 and goes on with a zero amplitude and no run (:659-668)
                        const uint32_t run = (sz > 1) ? 0u : ((e >> 10) & 15u);
                        const uint32_t bits = r.get(eob ? run : (sz == 1 ? 1u : 0u));  // the sign of a new coefficient / the length of an EOB run
                        const int sign = (sz == 1) ? (bits ? 1 : -1) : 0;             // 0: nothing to place (ZRL, ignored sizes)
                        const unsigned long long ahead = band & ~((1ull << k) - 1ull);  // the band from k on
                        // the (run+1)-th zero position at or behind k inside the band: whole low word first (one population
                        // count), then bit by bit in ONE 32-bit word -- two instructions per skipped position; the lanes of a
                        // warp run this loop together, as long as the longest run among them
                        const unsigned long long zeros = ~H & ahead;
                        uint32_t zw = (uint32_t)zeros, zbase = 0u, zn = eob ? 0u : run;
                        {
                            const uint32_t c = (uint32_t)__popc(zw);
                            if (zn >= c) zn -= c, zw = (uint32_t)(zeros >> 32), zbase = 32u;
                        }
#pragma unroll 2
                        for (uint32_t i = 0; i < zn; i++) zw &= zw - 1u;
                        const int target = (zw && !eob) ? (int)zbase + __ffs((int)zw) - 1 : se + 1;
                        const unsigned long long upto = (target >= 64) ? ~0ull : ((1ull << target) - 1ull);
                        if ((int)e < 0) {
                            bad = true;
                            active = false;
                        } else {
                            pending = H & ahead & upto;  // EOBn: target = se + 1, the whole rest of the band
                            if (target <= se && sign) {  // (its position is behind every position that still owes a bit)
                                uint2 pq;
                                asm("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(pq.x), "=r"(pq.y) : "r"(qz + 8u * (uint32_t)target));
                                const int d = sign * (int)pq.x;
                                ovf |= (uint32_t)(d + 32768);
                                sts_h(s_stage + pq.y, d);
                                H |= 1ull << target;
                            }
                            if (eob) {  // the rest of this block (and of the next skip-1 blocks) only takes correction bits
                                run_left = (1u << run) | bits;
                                tail = true;
                            }
                            k = target + 1;
                            if (eob || k > se) active = false;
                        }
                    }
                    if (pending != 0ull) {
                        const int p = __ffsll((long long)pending) - 1;
                        pending &= pending - 1ull;
                        if (r.get(1)) {
                            uint2 pq;
                            asm("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(pq.x), "=r"(pq.y) : "r"(qz + 8u * (uint32_t)p));
                            const int cur = lds_h(s_stage + pq.y);
                            const int d = cur + (cur > 0 ? (int)pq.x : -(int)pq.x);  // away from zero by 1 << Al, dequantised
                            ovf |= (uint32_t)(d + 32768);
                            sts_h(s_stage + pq.y, d);
                        }
                    }
                }
                if (tail && !bad) run_left--;
            }
            if (reads) s_park[(4 * s + 2) * kPfThreads] = r.bp;
            if (run_left != run_was) s_park[(4 * s + 3) * kPfThreads] = run_left;
        }
        if (has && !bad) {
            // ---- the DC value from the side plane, dequantised
            {
                const int level = L.dcplane[plane / 64u + (uint64_t)by * L.bw[0] + bx];
                const int d = level * dcq;
                ovf |= (uint32_t)(d + 32768);
                sts_h(s_stage, d);
            }
        }
        // ---- flush (zeros included) and clear the staging blocks, the whole warp together (see entropy_decode_kernel)
        {
            const int16_t *d = L.coef + plane + ((uint64_t)by * L.bw[0] + bx) * 64u;
            sts_q(s_stage + 136, has ? (uint64_t)d : 0ull);
            __syncwarp();
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const uint32_t a = s_flush + i * (4 * kStage);
                const uint64_t dst = lds_q(a + 136 - s_flush_sub);
                const uint4 v = lds16(a);
                sts_zero16(a);
                if (dst) *reinterpret_cast<uint4 *>(dst + s_flush_sub) = v;
            }
            __syncwarp();
        }
        if (++bx == L.mcu_cols) bx = 0, by++;
    }
    uint32_t err = 0;
    if (bad || (ovf >> 16) != 0u) err = kErrMalformed;
    if (err && lane_valid) atomicMax(L.frame_status + cs.frame, err);
}

}  // namespace

int launch_pf_dc(const PfLaunch &L, void *stream) {
    const uint64_t total = (uint64_t)L.n_frames * L.intervals;
    if (total == 0 || L.n_scans == 0) return 0;
    const size_t smem = (size_t)L.scan[0].lut_words * 4;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(pf_dc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    pf_dc_kernel<<<(uint32_t)((total + kPfThreads - 1) / kPfThreads), kPfThreads, smem, (cudaStream_t)stream>>>(L);
    return (int)cudaGetLastError();
}

int launch_pf_ac(const PfLaunch &L, void *stream) {
    const uint64_t total = (uint64_t)L.n_frames * L.intervals;
    if (total == 0 || L.n_scans == 0) return 0;
    size_t smem = (size_t)kPfThreads * kStage + (size_t)L.n_scans * 4 * kPfThreads * 4 + 2 * kPfMaxScans * 4;
    for (int s = 0; s < L.n_scans; s++) smem += (128u + (L.scan[s].lut_share == s ? (size_t)L.scan[s].lut_words : 0u)) * 4;
    if (smem > 227 * 1024) return (int)cudaErrorInvalidValue;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(pf_ac_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
    }
    pf_ac_kernel<<<(uint32_t)((total + kPfThreads - 1) / kPfThreads), kPfThreads, smem, (cudaStream_t)stream>>>(L);
    return (int)cudaGetLastError();
}

}  // namespace b200jpg
