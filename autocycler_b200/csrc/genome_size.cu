// Device part of `autocycler helper genome_size`: the reads packed to 2 bits per base, their canonical k-mers counted in partitions of
// an open-addressing table, and the histogram of the counts.  The reference runs an assembler here (helper.rs:388-403); this estimate
// comes from the reads' k-mer depth spectrum instead (DESIGN.md §18).  This file compiles with nvcc for sm_90a (product) and with
// g++ -DAC_EMULATE (tests/emu, serial execution of the same bodies).
#include "commands.h"
#include "gs_kmers.h"

#include <algorithm>
#include <stdexcept>
#include <utility>

// ------------------------------------------------------------------------------------------------
// genome_size: pack, count and histogram, see DESIGN.md §18
// ------------------------------------------------------------------------------------------------
// The packed stream: word w holds 32 bases, base i in bits 2i..2i+1 of code[w] (A=0, C=1, G=2, T=3; any other byte 0) and bit i of
// valid[w] set when the byte was A, C, G or T in either case.  Record r takes seq_len / 32 + 1 words, so at least one invalid base
// follows every read and no window of valid bases crosses into the next.

struct GsWordsBody {                                // record r's words; size[R] stays 0 for the scan's total
    const SubRecord* rec; uint64_t* size;
    AC_D void operator()(uint64_t r) const { size[r] = rec[r].seq_len / 32 + 1; }
};
// One warp of threads per record: lane l packs words l, l + 32, ... and counts the windows that end in them (it rebuilds word w-1's
// mask from the bytes, so no lane waits for another).  tot[0] += windows, tot[1] += bases.
struct GsPackBody {
    const uint8_t* bytes; const SubRecord* rec; const uint64_t* woff; uint64_t base; uint32_t k; uint64_t* code; uint32_t* valid; uint64_t* tot;
    AC_D void operator()(uint64_t t) const {
        const uint64_t r = t >> 5, lane = t & 31;
        const SubRecord o = rec[r];
        const uint8_t* s = bytes + o.seq;
        const uint64_t nw = o.seq_len / 32 + 1, w0 = base + woff[r];
        uint64_t windows = 0;
        for (uint64_t w = lane; w < nw; w += 32) {
            uint64_t c;
            const uint32_t v = gs_pack_word(s, o.seq_len, w, &c);
            const uint32_t pv = w ? gs_pack_word(s, o.seq_len, w - 1, nullptr) : 0;
            code[w0 + w] = c;
            valid[w0 + w] = v;
            windows += ac_popc(gs_window_ends(v, pv, k));
        }
        if (windows) ac_atomic_add(tot, windows);
        if (lane == 0 && o.seq_len) ac_atomic_add(tot + 1, (uint64_t)o.seq_len);
    }
};
// One thread per packed word: the forward and reverse keys roll over word w-1's last k-1 bases and then w's 32; each window that ends
// in w and whose canonical key falls in partition `part` of `parts` is counted.  Linear probing from the home slot; a key is claimed
// with a CAS on the empty slot.  The count is added only while a plain read shows it below 2^31, so it cannot wrap (the adds that race
// past the check are bounded by the resident threads).  After `limit` probes the window is dropped and *overflow set: the partition is
// counted again with more slots.
struct GsCountBody {
    const uint64_t* code; const uint32_t* valid; uint32_t k; uint64_t parts, part; GsSlot* table; uint64_t slots, limit; uint32_t* overflow;
    AC_D void operator()(uint64_t w) const {
        const uint32_t ends = gs_window_ends(valid[w], w ? valid[w - 1] : 0, k);
        if (!ends) return;
        const uint64_t c = code[w], pc = w ? code[w - 1] : 0, mask = (1ull << (2 * k)) - 1;
        const uint32_t top = 2 * (k - 1);
        uint64_t f = 0, rc = 0;
        for (uint32_t i = 32 - (k - 1); i < 32; ++i) {
            const uint64_t b = (pc >> (2 * i)) & 3;
            f = ((f << 2) | b) & mask; rc = (rc >> 2) | ((3 - b) << top);
        }
        for (uint32_t i = 0; i < 32; ++i) {
            const uint64_t b = (c >> (2 * i)) & 3;
            f = ((f << 2) | b) & mask; rc = (rc >> 2) | ((3 - b) << top);
            if (!((ends >> i) & 1)) continue;
            const uint64_t key = f < rc ? f : rc, h = gs_mix(key);
            if (ac_umul64hi(h, parts) != part) continue;
            uint64_t s = ac_umul64hi(h * parts, slots);
            const uint64_t tag = key + 1;
            bool done = false;
            for (uint64_t n = 0; n < limit && !done; ++n) {
                GsSlot* q = table + s;
                uint64_t cur = ac_ld_volatile(&q->key);
                if (cur == 0) cur = ac_atomic_cas(&q->key, (uint64_t)0, tag);
                if (cur == 0 || cur == tag) {
                    if (ac_ld_volatile(&q->count) < 0x80000000u) ac_atomic_add(&q->count, 1u);
                    done = true;
                } else if (++s == slots) s = 0;
            }
            if (!done) ac_atomic_max(overflow, 1u);
        }
    }
};
AC_HD uint32_t gs_bin(const GsSlot& q) {                    // 0: an empty slot
    return q.key ? (q.count < AC_GS_BINS - 1 ? q.count : AC_GS_BINS - 1) : 0;
}

#ifndef AC_EMULATE
// One thread per slot; each CTA counts into a shared-memory copy of the bins (64 KiB of u32) and adds its non-zero bins to the
// global u64 histogram once.
__global__ void __launch_bounds__(1024) ac_gs_hist_kernel(const GsSlot* __restrict__ table, uint64_t slots, unsigned long long* hist) {
    extern __shared__ uint32_t gs_bins[];
    for (uint32_t i = threadIdx.x; i < AC_GS_BINS; i += blockDim.x) gs_bins[i] = 0;
    __syncthreads();
    for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < slots; s += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t b = gs_bin(table[s]);
        if (b) atomicAdd(gs_bins + b, 1u);
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < AC_GS_BINS; i += blockDim.x)
        if (gs_bins[i]) atomicAdd(hist + i, (unsigned long long)gs_bins[i]);
}
#else
struct GsHistBody {                                 // the same, one slot at a time
    const GsSlot* table; uint64_t* hist;
    void operator()(uint64_t s) const { const uint32_t b = gs_bin(table[s]); if (b) ++hist[b]; }
};
#endif

namespace {
void grow_keep(DevBuf& b, size_t want, size_t keep, AcStream* st) {     // device memory that keeps its first `keep` bytes
    if (want <= b.cap) return;
    DevBuf nb;
    nb.ensure(std::max(want, 2 * b.cap));
    if (keep) ac_copy_dd(nb.p, b.p, keep, st);
    ac_sync(st);
    std::swap(b.p, nb.p); std::swap(b.cap, nb.cap);
}
}  // namespace

uint64_t ac_gs_budget_slots() {
#ifdef AC_EMULATE
    return 1ull << 25;
#else
    size_t free_b = 0, total_b = 0;
    AC_CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
    return (uint64_t)(free_b / 2) / sizeof(GsSlot);
#endif
}

void DeviceSpectrum::begin(uint32_t kk) {
    ctx.make_current();
    k = kk; words = 0; kernel_ms = 0.f; pack_ms = 0.f;
    part_slots.clear();
    d_tot.ensure(16);
    ac_memset(d_tot.p, 0, 16, &ctx.stream);
}

void DeviceSpectrum::pack_window(DeviceSubsample& sub, uint64_t R) {
    if (!R) return;
    ctx.make_current();
    AcStream* st = &ctx.stream;
    d_woff.ensure((R + 1) * 8);
    uint64_t* woff = d_woff.as<uint64_t>();
    ac_memset(woff + R, 0, 8, st);
    AcTimer timer(st);
    ac_launch("gs_words", st, GsWordsBody{sub.window_records(), woff}, R);
    const uint64_t n = scan_u64.run(st, woff, woff, R + 1, true);
    timer.stop();
    ac_sync(st);
    pack_ms += timer.ms();
    grow_keep(d_code, (words + n) * 8, words * 8, st);
    grow_keep(d_valid, (words + n) * 4, words * 4, st);
    AcTimer t2(st);
    ac_launch("gs_pack", st, GsPackBody{sub.window_bytes(), sub.window_records(), woff, words, k, d_code.as<uint64_t>(), d_valid.as<uint32_t>(),
                                        d_tot.as<uint64_t>()}, R * 32);
    t2.stop();
    ac_sync(st);
    pack_ms += t2.ms();
    words += n;
}

void DeviceSpectrum::totals(uint64_t* windows, uint64_t* bases) {
    ctx.make_current();
    uint64_t t[2];
    ac_d2h(t, d_tot.p, 16, &ctx.stream);
    ac_sync(&ctx.stream);
    *windows = t[0]; *bases = t[1];
}

// One partition's table in d_table: counted at `slots` slots, and again at twice the slots while the probe limit is hit.  Returns the
// slot count that held it.
uint64_t DeviceSpectrum::count_partition(uint64_t parts, uint64_t part, uint64_t slots, SpectrumRun* run) {
    AcStream* st = &ctx.stream;
    for (;; slots *= 2) {
        if (slots > (1ull << 40)) throw std::runtime_error("genome_size: the k-mer table cannot hold one partition");
        d_table.ensure(slots * sizeof(GsSlot));
        run->table_bytes = std::max<uint64_t>(run->table_bytes, slots * sizeof(GsSlot));
        GsSlot* table = d_table.as<GsSlot>();
        ac_memset(table, 0, slots * sizeof(GsSlot), st);
        ac_memset(d_flag.p, 0, 4, st);
        const uint64_t limit = std::min<uint64_t>(slots, 4096);
        AcTimer tc(st);
        ac_launch("gs_count", st, GsCountBody{d_code.as<uint64_t>(), d_valid.as<uint32_t>(), k, parts, part, table, slots, limit,
                                              d_flag.as<uint32_t>()}, words);
        tc.stop();
        uint32_t overflow = 0;
        ac_d2h(&overflow, d_flag.p, 4, st);
        ac_sync(st);
        run->count_ms += tc.ms();
        if (overflow) { ++run->reruns; continue; }
        resident = part;
        return slots;
    }
}

void DeviceSpectrum::count(uint64_t W, uint64_t budget, uint64_t parts, uint64_t* hist, SpectrumRun* run) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    *run = SpectrumRun();
    run->pack_ms = pack_ms;
    if (budget < 1) budget = 1;
    const uint64_t want = 2 * W;
    if (!parts) { parts = 1; while ((want + parts - 1) / parts > budget) parts *= 2; }
    const uint64_t base_slots = std::max<uint64_t>(1, std::min((want + parts - 1) / parts, budget));
    d_hist.ensure(AC_GS_BINS * 8); d_flag.ensure(4);
    ac_memset(d_hist.p, 0, AC_GS_BINS * 8, st);
    part_slots.clear();
    for (uint64_t part = 0; part < parts; ++part) {
        const uint64_t slots = count_partition(parts, part, base_slots, run);
        part_slots.push_back(slots);
        const GsSlot* table = d_table.as<GsSlot>();
        AcTimer th(st);
#ifndef AC_EMULATE
        const uint64_t blocks = std::min<uint64_t>((slots + 1023) / 1024, 2 * ac_sm_count());
        ac_launch_kernel("gs_hist", st, ac_gs_hist_kernel, (unsigned)blocks, 1024, AC_GS_BINS * 4, table, slots,
                         d_hist.as<unsigned long long>());
#else
        ac_launch("gs_hist", st, GsHistBody{table, d_hist.as<uint64_t>()}, slots);
#endif
        th.stop();
        ac_sync(st);
        run->hist_ms += th.ms();
    }
    ac_d2h(hist, d_hist.p, AC_GS_BINS * 8, st);
    ac_sync(st);
    run->partitions = parts;
    kernel_ms = run->pack_ms + run->count_ms + run->hist_ms;
}

void DeviceSpectrum::sweep(const std::function<void(const GsSlot*, uint64_t, uint64_t, uint64_t)>& each, SpectrumRun* run) {
    ctx.make_current();
    const uint64_t parts = part_slots.size();
    if (!parts) throw std::logic_error("genome_size: a second sweep before the count");
    // the partition whose table is still in d_table goes first; every other one is counted again at its settled slots
    const uint64_t first = resident;
    for (uint64_t i = 0; i < parts; ++i) {
        const uint64_t part = (first + i) % parts;
        uint64_t slots = part_slots[part];
        if (i) slots = count_partition(parts, part, slots, run);
        each(d_table.as<GsSlot>(), slots, parts, part);
    }
    run->partitions = parts;
}
