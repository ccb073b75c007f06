// Device part of `autocycler depth`: the assembly's canonical k-mers in one open-addressing table, the reads' packed stream probed
// against it, and each contig's exact median count selected on the device.  Read-measured depth is not in the reference; only the
// filter on the depths (host_depth.cpp) is.  This file compiles with nvcc for sm_90a (product) and with g++ -DAC_EMULATE (tests/emu,
// serial execution of the same bodies).
#include "commands.h"
#include "dp_kmers.h"

#include <algorithm>
#include <cmath>
#include <stdexcept>
#include <vector>

// ------------------------------------------------------------------------------------------------
// depth: pack, insert, probe and median, see DESIGN.md §19
// ------------------------------------------------------------------------------------------------
namespace {
// One thread per packed word of the assembly: each window's key is inserted by linear probing from its home slot, claimed with a CAS
// on the empty key.  The claimer ORs its contig id into the flags; every later occurrence ORs AC_DEPTH_DUP.  The table holds at least
// twice the windows, so a probe always finds its key or an empty slot.
struct DpInsertBody {
    const uint64_t* code; const uint32_t* valid; const uint32_t* wcid; uint32_t k; DepthSlot* table; uint64_t slots;
    AC_D void operator()(uint64_t w) const {
        dp_each_key(code, valid, w, k, [&](uint64_t key) {
            uint64_t s = ac_umul64hi(gs_mix(key), slots);
            const uint64_t tag = key + 1;
            for (;;) {
                DepthSlot* q = table + s;
                uint64_t cur = ac_ld_volatile(&q->key);
                if (cur == 0) cur = ac_atomic_cas(&q->key, (uint64_t)0, tag);
                if (cur == 0) { ac_atomic_or(&q->flags, wcid[w]); return; }
                if (cur == tag) { ac_atomic_or(&q->flags, AC_DEPTH_DUP); return; }
                if (++s == slots) s = 0;
            }
        });
    }
};
AC_HD bool dp_unique(const DepthSlot& q) { return q.key && !(q.flags & AC_DEPTH_DUP); }
// One thread per slot: unique[contig] += 1 for a unique key.
struct DpUniqueBody {
    const DepthSlot* table; uint32_t* unique;
    AC_D void operator()(uint64_t s) const { const DepthSlot q = table[s]; if (dp_unique(q)) dp_add_one(unique + q.flags); }
};
// One thread per contig: the ranks of its lower and upper middle counts, (n-1)/2 and n/2, and empty prefixes.
struct DpRankBody {
    const uint32_t* unique; uint32_t* rank; uint32_t* prefix;
    AC_D void operator()(uint64_t c) const {
        const uint32_t n = unique[c];
        rank[2 * c] = n ? (n - 1) / 2 : 0; rank[2 * c + 1] = n / 2;
        prefix[2 * c] = 0; prefix[2 * c + 1] = 0;
    }
};
// One radix-select pass over the slots, digit (count >> shift) & 255: a unique key whose count agrees with the selection's prefix above
// the digit adds 1 to hist[(2 contig + r) * 256 + digit], for the lower (r = 0) and upper (r = 1) middle.
struct DpDigitBody {
    const DepthSlot* table; const uint32_t* prefix; uint32_t shift; uint32_t* hist;
    AC_D void operator()(uint64_t s) const {
        const DepthSlot q = table[s];
        if (!dp_unique(q)) return;
        const uint32_t d = (q.count >> shift) & 255u;
        for (uint32_t r = 0; r < 2; ++r) {
            const uint64_t i = 2 * (uint64_t)q.flags + r;
            if ((((uint64_t)(q.count ^ prefix[i])) >> (shift + 8)) == 0) dp_add_one(hist + i * 256 + d);
        }
    }
};
// One thread per (contig, r): the digit that holds rank[i] joins the prefix, and the rank becomes the rank within that digit.
struct DpSelectBody {
    const uint32_t* unique; const uint32_t* hist; uint32_t shift; uint32_t* rank; uint32_t* prefix;
    AC_D void operator()(uint64_t i) const {
        if (!unique[i / 2]) return;
        uint32_t r = rank[i];
        for (uint32_t d = 0; d < 256; ++d) {
            const uint32_t h = hist[i * 256 + d];
            if (r < h) { prefix[i] |= d << shift; rank[i] = r; return; }
            r -= h;
        }
    }
};
// One thread per contig: the median, the mean of the two middle counts in f64 (exact), NaN without unique keys.
struct DpMedianBody {
    const uint32_t* unique; const uint32_t* prefix; double* median;
    AC_D void operator()(uint64_t c) const {
        median[c] = unique[c] ? ((double)prefix[2 * c] + (double)prefix[2 * c + 1]) / 2.0 : NAN;
    }
};
}  // namespace

void DeviceDepth::build(const uint8_t* bytes, const uint64_t* len, uint32_t n, uint64_t windows, uint32_t kk, uint64_t budget, DepthRun* run) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    if (n >= AC_DEPTH_DUP) throw std::length_error("depth: an assembly of 2^31 contigs or more");
    k = kk; n_contigs = n;
    slots = std::max<uint64_t>(2 * windows, 64);
    run->assembly_windows = windows;
    run->table_bytes = slots * sizeof(DepthSlot);
    if (slots > budget)
        throw std::length_error("depth: the assembly's k-mer table (" + std::to_string(run->table_bytes) + " bytes) does not fit half the free device memory");
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
    ac_launch("dp_pack", st, DpPackBody{d_bytes.as<uint8_t>(), d_contig.as<DpContig>(), n, d_code.as<uint64_t>(), d_valid.as<uint32_t>(),
                                        d_wcid.as<uint32_t>()}, words);
    tp.stop();
    AcTimer ti(st);
    ac_launch("dp_insert", st, DpInsertBody{d_code.as<uint64_t>(), d_valid.as<uint32_t>(), d_wcid.as<uint32_t>(), k, d_table.as<DepthSlot>(),
                                            slots}, words);
    ti.stop();
    ac_sync(st);
    run->pack_ms += tp.ms(); run->insert_ms += ti.ms();
}

void DeviceDepth::probe(DeviceSpectrum& spec, DepthRun* run) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    AcTimer t(st);
    ac_launch("dp_probe", st, DpProbeBody{spec.packed_codes(), spec.packed_valid(), k, d_table.as<DepthSlot>(), slots}, spec.packed_words());
    t.stop();
    ac_sync(st);
    run->probe_ms += t.ms();
}

void DeviceDepth::medians(uint64_t* unique, double* median, DepthRun* run) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    const uint64_t n = n_contigs;
    if (!n) return;
    d_unique.ensure(n * 4); d_rank.ensure(n * 8); d_prefix.ensure(n * 8); d_hist.ensure(n * 2 * 256 * 4); d_median.ensure(n * 8);
    uint32_t* u = d_unique.as<uint32_t>(), *rank = d_rank.as<uint32_t>(), *prefix = d_prefix.as<uint32_t>(), *hist = d_hist.as<uint32_t>();
    const DepthSlot* table = d_table.as<DepthSlot>();
    ac_memset(u, 0, n * 4, st);
    AcTimer t(st);
    ac_launch("dp_unique", st, DpUniqueBody{table, u}, slots);
    ac_launch("dp_rank", st, DpRankBody{u, rank, prefix}, n);
    for (int shift = 24; shift >= 0; shift -= 8) {                  // four 8-bit digits of the u32 count, the highest first
        ac_memset(hist, 0, n * 2 * 256 * 4, st);
        ac_launch("dp_digit", st, DpDigitBody{table, prefix, (uint32_t)shift, hist}, slots);
        ac_launch("dp_select", st, DpSelectBody{u, hist, (uint32_t)shift, rank, prefix}, 2 * n);
    }
    ac_launch("dp_median", st, DpMedianBody{u, prefix, d_median.as<double>()}, n);
    t.stop();
    std::vector<uint32_t> h_unique(n);
    ac_d2h(h_unique.data(), u, n * 4, st);
    ac_d2h(median, d_median.p, n * 8, st);
    ac_sync(st);
    for (uint64_t c = 0; c < n; ++c) unique[c] = h_unique[c];
    run->median_ms += t.ms();
}
