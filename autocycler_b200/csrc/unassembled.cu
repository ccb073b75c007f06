// Device part of `autocycler unassembled`: the assembly's canonical k-mers claimed in one table, each packed read word tagged with its
// read, and a second sweep over the read spectrum's partitions that counts, per read, its solid windows and those the assembly lacks,
// and bins the solid keys the assembly lacks.  Not in the reference (DESIGN.md §21).  This file compiles with nvcc for sm_90a (product)
// and with g++ -DAC_EMULATE (tests/emu, serial execution of the same bodies).
#include "commands.h"
#include "dp_kmers.h"

#include <algorithm>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

// ------------------------------------------------------------------------------------------------
// unassembled: pack, claim, index, then the attribution sweep, see DESIGN.md §21
// ------------------------------------------------------------------------------------------------
namespace {
// One warp per record of the window just packed: lane l writes the read's index into the record's packed words l, l + 32, ...; lane 0
// writes its sequence length.
struct UaIndexBody {
    const SubRecord* rec; const uint64_t* woff; uint64_t word0, first; uint32_t* read; uint32_t* len;
    AC_D void operator()(uint64_t t) const {
        const uint64_t r = t >> 5, lane = t & 31, w0 = word0 + woff[r], nw = woff[r + 1] - woff[r];
        for (uint64_t w = lane; w < nw; w += 32) read[w0 + w] = (uint32_t)(first + r);
        if (lane == 0) len[first + r] = rec[r].seq_len;
    }
};
// *p += s | a << 32 (the read's two u32 counters; s < 2^32 for any read).  On the device the lanes of a warp that add to the same read
// are grouped first, one atomic per group: consecutive words almost always belong to one read.
#ifdef AC_EMULATE
inline void ua_add(uint64_t* p, uint32_t s, uint32_t a) { *p += s | (uint64_t)a << 32; }
#else
__device__ __forceinline__ void ua_add(uint64_t* p, uint32_t s, uint32_t a) {
    const unsigned same = __match_any_sync(__activemask(), (unsigned long long)p);
    s = __reduce_add_sync(same, s);
    a = __reduce_add_sync(same, a);
    if ((int)(threadIdx.x & 31) == __ffs((int)same) - 1) atomicAdd((unsigned long long*)p, (unsigned long long)s | (unsigned long long)a << 32);
}
#endif
// One thread per packed read word, for the windows whose key falls in partition `part`: a window whose key the reads hold t times or
// more adds 1 to its read's s, and also to its a when the assembly set does not hold the key.
struct UaAttributeBody {
    const uint64_t* code; const uint32_t* valid; const uint32_t* read; uint32_t k; uint64_t parts, part; const GsSlot* spec; uint64_t spec_slots;
    const DepthSlot* table; uint64_t slots; uint32_t t; uint64_t* counts;
    AC_D void operator()(uint64_t w) const {
        uint32_t s = 0, a = 0;
        dp_each_key(code, valid, w, k, [&](uint64_t key) {
            const uint64_t h = gs_mix(key);
            if (ac_umul64hi(h, parts) != part || ua_read_count(spec, spec_slots, parts, h, key) < t) return;
            ++s;
            if (!dp_holds(table, slots, key)) ++a;
        });
        if (s) ua_add(counts + read[w], s, a);
    }
};
// One thread per slot of a partition's table: a key the reads hold t times or more and the assembly set does not adds 1 to its bin.
struct UaAbsentBody {
    const GsSlot* spec; const DepthSlot* table; uint64_t slots; uint32_t t; uint32_t* absent;
    AC_D void operator()(uint64_t s) const {
        const GsSlot q = spec[s];
        if (!q.key || q.count < t || dp_holds(table, slots, q.key - 1)) return;
        dp_add_one(absent + (q.count < AC_GS_BINS - 1 ? q.count : AC_GS_BINS - 1));
    }
};

void grow_keep(DevBuf& b, size_t want, size_t keep, AcStream* st) {     // device memory that keeps its first `keep` bytes
    if (want <= b.cap) return;
    DevBuf nb;
    nb.ensure(std::max(want, 2 * b.cap));
    if (keep) ac_copy_dd(nb.p, b.p, keep, st);
    ac_sync(st);
    std::swap(b.p, nb.p); std::swap(b.cap, nb.cap);
}
}  // namespace

void DeviceUnassembled::build(const uint8_t* bytes, const uint64_t* len, uint32_t n, uint64_t windows, uint32_t kk, uint64_t budget, UaRun* run) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    k = kk;
    slots = std::max<uint64_t>(2 * windows, 64);
    run->assembly_windows = windows;
    run->table_bytes = slots * sizeof(DepthSlot);
    if (slots > budget)
        throw std::length_error("unassembled: the assembly's k-mer table (" + std::to_string(run->table_bytes) + " bytes) does not fit half the free device memory");
    std::vector<DpContig> contig(n + 1);
    uint64_t off = 0, words = 0;
    for (uint32_t c = 0; c < n; ++c) {
        contig[c] = DpContig{off, len[c], words};
        off += len[c]; words += len[c] / 32 + 1;
    }
    contig[n] = DpContig{off, 0, words};
    d_bytes.ensure(std::max<uint64_t>(off, 1)); d_contig.ensure((n + 1) * sizeof(DpContig));
    d_code.ensure(words * 8); d_valid.ensure(words * 4); d_wcid.ensure(words * 4);
    d_table.ensure(slots * sizeof(DepthSlot));
    if (off) ac_h2d(d_bytes.p, bytes, off, st);
    ac_h2d(d_contig.p, contig.data(), (n + 1) * sizeof(DpContig), st);
    ac_memset(d_table.p, 0, slots * sizeof(DepthSlot), st);
    AcTimer tp(st);
    ac_launch("ua_pack", st, DpPackBody{d_bytes.as<uint8_t>(), d_contig.as<DpContig>(), n, d_code.as<uint64_t>(), d_valid.as<uint32_t>(),
                                        d_wcid.as<uint32_t>()}, words);
    tp.stop();
    AcTimer tc(st);
    ac_launch("ua_claim", st, QvClaimBody{d_code.as<uint64_t>(), d_valid.as<uint32_t>(), k, d_table.as<DepthSlot>(), slots}, words);
    tc.stop();
    ac_sync(st);
    run->pack_ms += tp.ms(); run->claim_ms += tc.ms();
}

void DeviceUnassembled::index_window(DeviceSpectrum& spec, DeviceSubsample& sub, uint64_t first, uint64_t records, uint64_t word0, UaRun* run) {
    if (!records) return;
    ctx.make_current();
    AcStream* st = &ctx.stream;
    grow_keep(d_read, spec.packed_words() * 4, word0 * 4, st);
    grow_keep(d_len, (first + records) * 4, first * 4, st);
    AcTimer timer(st);
    ac_launch("ua_index", st, UaIndexBody{sub.window_records(), spec.window_word_offsets(), word0, first, d_read.as<uint32_t>(),
                                          d_len.as<uint32_t>()}, records * 32);
    timer.stop();
    ac_sync(st);
    run->index_ms += timer.ms();
}

void DeviceUnassembled::check_budget(uint64_t reads, uint64_t words, uint64_t budget, UaRun* run) {
    run->read_bytes = 12 * reads + 4 * words;                  // s and a, the length, per read; the read index per packed word
    if (run->table_bytes + run->read_bytes > budget * sizeof(GsSlot))
        throw std::length_error("unassembled: the assembly's k-mer table and the per-read counters (" +
                                std::to_string(run->table_bytes + run->read_bytes) + " bytes) do not fit half the free device memory");
}

void DeviceUnassembled::attribute(DeviceSpectrum& spec, uint64_t reads, uint32_t t, uint32_t* counts, uint32_t* lengths, uint64_t* absent,
                                  UaRun* run) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    d_counts.ensure(std::max<uint64_t>(reads, 1) * 8); d_absent.ensure(AC_GS_BINS * 4);
    ac_memset(d_counts.p, 0, std::max<uint64_t>(reads, 1) * 8, st);
    ac_memset(d_absent.p, 0, AC_GS_BINS * 4, st);
    run->sweep = SpectrumRun();
    spec.sweep([&](const GsSlot* table, uint64_t spec_slots, uint64_t parts, uint64_t part) {
        AcTimer timer(st);
        ac_launch("ua_attribute", st, UaAttributeBody{spec.packed_codes(), spec.packed_valid(), d_read.as<uint32_t>(), k, parts, part, table,
                                                      spec_slots, d_table.as<DepthSlot>(), slots, t, d_counts.as<uint64_t>()},
                  spec.packed_words());
        ac_launch("ua_absent", st, UaAbsentBody{table, d_table.as<DepthSlot>(), slots, t, d_absent.as<uint32_t>()}, spec_slots);
        timer.stop();
        ac_sync(st);
        run->attribute_ms += timer.ms();
    }, &run->sweep);
    std::vector<uint32_t> bins(AC_GS_BINS);
    if (reads) { ac_d2h(counts, d_counts.p, reads * 8, st); ac_d2h(lengths, d_len.p, reads * 4, st); }
    ac_d2h(bins.data(), d_absent.p, AC_GS_BINS * 4, st);
    ac_sync(st);
    for (uint32_t c = 0; c < AC_GS_BINS; ++c) absent[c] = bins[c];
}
