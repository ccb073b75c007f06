// Device part of `autocycler qv`: every assembly's canonical k-mers claimed in one combined table, the reads' packed stream probed
// against it once, then per assembly a multiplicity table, a mask of its unsupported windows and its copy-number spectrum.  Not in the
// reference (DESIGN.md §20).  This file compiles with nvcc for sm_90a (product) and with g++ -DAC_EMULATE (tests/emu, serial execution
// of the same bodies).
#include "commands.h"
#include "dp_kmers.h"

#include <algorithm>
#include <stdexcept>
#include <string>
#include <vector>

// ------------------------------------------------------------------------------------------------
// qv: pack, claim, probe, then multiplicity, support and spectrum per assembly, see DESIGN.md §20
// ------------------------------------------------------------------------------------------------
namespace {
// One thread per packed word of one assembly (from word w0): each window adds 1 to its key's m in the multiplicity table; the thread
// that claims the slot copies the key's read count from the combined table.
struct QvMultBody {
    const uint64_t* code; const uint32_t* valid; uint32_t k; uint64_t w0; const DepthSlot* table; uint64_t slots; QvSlot* mult; uint64_t mslots;
    AC_D void operator()(uint64_t i) const {
        dp_each_key(code, valid, w0 + i, k, [&](uint64_t key) {
            uint64_t s = ac_umul64hi(gs_mix(key), mslots);
            const uint64_t tag = key + 1;
            for (;;) {
                QvSlot* q = mult + s;
                uint64_t cur = ac_ld_volatile(&q->key);
                if (cur == 0) cur = ac_atomic_cas(&q->key, (uint64_t)0, tag);
                if (cur == 0) q->r = qv_read_count(table, slots, key);
                if (cur == 0 || cur == tag) { ac_atomic_add(&q->m, 1u); return; }
                if (++s == mslots) s = 0;
            }
        });
    }
};
// One thread per packed word of one assembly: bit j of mask[i] is set when the window that ends at base j has a read count below t.
struct QvSupportBody {
    const uint64_t* code; const uint32_t* valid; uint32_t k; uint64_t w0; const QvSlot* mult; uint64_t mslots; uint32_t t; uint32_t* mask;
    AC_D void operator()(uint64_t i) const {
        const uint64_t w = w0 + i;
        uint32_t rest = gs_window_ends(valid[w], w ? valid[w - 1] : 0, k), bits = 0;     // dp_each_key visits these ends, lowest first
        dp_each_key(code, valid, w, k, [&](uint64_t key) {
            const uint32_t bit = rest & (0u - rest);
            rest ^= bit;
            uint64_t s = ac_umul64hi(gs_mix(key), mslots);
            for (;;) {
                const QvSlot* q = mult + s;
                if (q->key == key + 1) { if (q->r < t) bits |= bit; return; }
                if (++s == mslots) s = 0;
            }
        });
        mask[i] = bits;
    }
};
// One thread per slot of the multiplicity table: spectrum[min(r, H - 1) * AC_QV_CN + min(m, 4)] += 1 for each key.
struct QvSpectrumBody {
    const QvSlot* mult; uint32_t* spectrum;
    AC_D void operator()(uint64_t s) const {
        const QvSlot q = mult[s];
        if (!q.key) return;
        const uint32_t c = q.r < AC_GS_BINS - 1 ? q.r : AC_GS_BINS - 1, m = q.m < 4 ? q.m : 4;
        dp_add_one(spectrum + (uint64_t)c * AC_QV_CN + m);
    }
};
}  // namespace

void DeviceQv::build(const uint8_t* bytes, const uint64_t* len, uint32_t n, const uint32_t* first, uint32_t n_assemblies,
                     const uint64_t* windows, uint32_t kk, uint64_t budget, QvRun* run) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    k = kk;
    uint64_t total = 0, largest = 0, largest_words = 0;
    woff.assign(n + 1, 0);
    std::vector<DpContig> contig(n + 1);
    uint64_t off = 0;
    for (uint32_t c = 0; c < n; ++c) {
        contig[c] = DpContig{off, len[c], woff[c]};
        off += len[c]; woff[c + 1] = woff[c] + len[c] / 32 + 1;
    }
    contig[n] = DpContig{off, 0, woff[n]};
    first_contig.assign(first, first + n_assemblies + 1);
    win.assign(windows, windows + n_assemblies);
    for (uint32_t a = 0; a < n_assemblies; ++a) {
        total += windows[a];
        largest = std::max(largest, windows[a]);
        largest_words = std::max(largest_words, woff[first[a + 1]] - woff[first[a]]);
    }
    slots = std::max<uint64_t>(2 * total, 64);
    mult_slots = std::max<uint64_t>(2 * largest, 64);
    run->assembly_windows = total;
    run->table_bytes = (slots + mult_slots) * sizeof(DepthSlot);
    if (slots + mult_slots > budget)
        throw std::length_error("qv: the assemblies' k-mer tables (" + std::to_string(run->table_bytes) + " bytes) do not fit half the free device memory");
    const uint64_t words = woff[n];
    d_bytes.ensure(std::max<uint64_t>(off, 1)); d_contig.ensure((n + 1) * sizeof(DpContig));
    d_code.ensure(words * 8); d_valid.ensure(words * 4); d_wcid.ensure(words * 4);
    d_table.ensure(slots * sizeof(DepthSlot)); d_mult.ensure(mult_slots * sizeof(QvSlot));
    d_mask.ensure(std::max<uint64_t>(largest_words, 1) * 4); d_spec.ensure((uint64_t)AC_GS_BINS * AC_QV_CN * 4);
    if (off) ac_h2d(d_bytes.p, bytes, off, st);
    ac_h2d(d_contig.p, contig.data(), (n + 1) * sizeof(DpContig), st);
    ac_memset(d_table.p, 0, slots * sizeof(DepthSlot), st);
    AcTimer tp(st);
    ac_launch("qv_pack", st, DpPackBody{d_bytes.as<uint8_t>(), d_contig.as<DpContig>(), n, d_code.as<uint64_t>(), d_valid.as<uint32_t>(),
                                        d_wcid.as<uint32_t>()}, words);
    tp.stop();
    AcTimer ti(st);
    ac_launch("qv_claim", st, QvClaimBody{d_code.as<uint64_t>(), d_valid.as<uint32_t>(), k, d_table.as<DepthSlot>(), slots}, words);
    ti.stop();
    ac_sync(st);
    run->pack_ms += tp.ms(); run->insert_ms += ti.ms();
}

void DeviceQv::probe(DeviceSpectrum& spec, QvRun* run) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    AcTimer t(st);
    ac_launch("qv_probe", st, DpProbeBody{spec.packed_codes(), spec.packed_valid(), k, d_table.as<DepthSlot>(), slots}, spec.packed_words());
    t.stop();
    ac_sync(st);
    run->probe_ms += t.ms();
}

void DeviceQv::assembly(uint32_t a, uint32_t t, uint32_t* mask, uint32_t* spectrum, QvRun* run) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    const uint64_t w0 = woff[first_contig[a]], words = woff[first_contig[a + 1]] - w0;
    const uint64_t ms = std::max<uint64_t>(2 * win[a], 64);
    QvSlot* mult = d_mult.as<QvSlot>();
    const uint64_t spec_bytes = (uint64_t)AC_GS_BINS * AC_QV_CN * 4;
    ac_memset(mult, 0, ms * sizeof(QvSlot), st);
    ac_memset(d_spec.p, 0, spec_bytes, st);
    AcTimer timer(st);
    ac_launch("qv_mult", st, QvMultBody{d_code.as<uint64_t>(), d_valid.as<uint32_t>(), k, w0, d_table.as<DepthSlot>(), slots, mult, ms}, words);
    ac_launch("qv_support", st, QvSupportBody{d_code.as<uint64_t>(), d_valid.as<uint32_t>(), k, w0, mult, ms, t, d_mask.as<uint32_t>()}, words);
    ac_launch("qv_spectrum", st, QvSpectrumBody{mult, d_spec.as<uint32_t>()}, ms);
    timer.stop();
    if (words) ac_d2h(mask, d_mask.p, words * 4, st);
    ac_d2h(spectrum, d_spec.p, spec_bytes, st);
    ac_sync(st);
    run->assembly_ms += timer.ms();
}
