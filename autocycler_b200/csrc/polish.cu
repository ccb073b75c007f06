// Device part of `autocycler polish`: each round's contigs packed and their canonical keys claimed in a query table whose read counts a
// sweep over the read spectrum's partitions fills, the mask of the windows the reads do not support, and for each attempted locus its
// candidate edits' checked windows claimed, filled, scored and reduced to a choice.  Not in the reference (DESIGN.md §22).  The fill, the
// candidates' windows, their claim and their score are in pl_kmers.h, which `variants` shares.  This file compiles with nvcc for sm_90a
// (product) and with g++ -DAC_EMULATE (tests/emu, serial execution of the same bodies).
#include "commands.h"
#include "dp_kmers.h"
#include "pl_kmers.h"

#include <algorithm>
#include <stdexcept>
#include <string>
#include <vector>

// ------------------------------------------------------------------------------------------------
// polish: pack, claim, fill and mask per round, then candidates, fill, score and choice per batch of loci, see DESIGN.md §22
// ------------------------------------------------------------------------------------------------
namespace {
// One thread per packed word of the round's contigs: bit j of mask[w] is set when the window that ends at base j has r < t.
struct PlSupportBody {
    const uint64_t* code; const uint32_t* valid; uint32_t k; const DepthSlot* table; uint64_t slots; uint32_t t; uint32_t* mask;
    AC_D void operator()(uint64_t w) const {
        uint32_t rest = gs_window_ends(valid[w], w ? valid[w - 1] : 0, k), bits = 0;     // dp_each_key visits these ends, lowest first
        dp_each_key(code, valid, w, k, [&](uint64_t key) {
            const uint32_t bit = rest & (0u - rest);
            rest ^= bit;
            if (qv_read_count(table, slots, key) < t) bits |= bit;
        });
        mask[w] = bits;
    }
};

AC_D void pl_take(uint32_t v, uint32_t c, uint32_t& best, uint32_t& count, uint32_t& first) {
    if (v > best) { best = v; count = 1; first = c; }
    else if (v && v == best) ++count;
}
// One warp per locus: out[3 l] = the best score (0: none passes), out[3 l + 1] = the candidates that hold it, out[3 l + 2] = the first.
struct PlChooseBody {
    const uint32_t* score; uint32_t C; uint32_t* out;
    AC_D void operator()(uint64_t t) const {
        const uint64_t l = t >> 5;
        const uint32_t lane = (uint32_t)(t & 31), * s = score + l * C;
        uint32_t best = 0, count = 0, first = 0;
#ifdef AC_EMULATE
        if (lane) return;
        for (uint32_t c = 0; c < C; ++c) pl_take(s[c], c, best, count, first);
#else
        for (uint32_t c = lane; c < C; c += 32) pl_take(s[c], c, best, count, first);
        // Every lane of the warp gets here (the launch is 32 threads per locus), but after the loop above, whose trip count differs
        // between lanes when C is not a multiple of 32, __activemask() need not name them all: the reductions take the whole warp.
        const unsigned all = 0xFFFFFFFFu;
        const uint32_t top = __reduce_max_sync(all, best);
        count = __reduce_add_sync(all, best == top ? count : 0u);
        first = __reduce_min_sync(all, best == top ? first : 0xFFFFFFFFu);
        best = top;
        if (lane) return;
#endif
        out[3 * l] = best; out[3 * l + 1] = best ? count : 0; out[3 * l + 2] = best ? first : 0;
    }
};
}  // namespace

uint64_t DevicePolish::candidates(uint32_t L) {
    uint64_t c = 3 + L, p = 1;
    for (uint32_t s = 1; s <= L; ++s) { p *= 4; c += p; }
    return c;
}

uint64_t DevicePolish::candidate_windows(uint32_t k, uint32_t L) {
    uint64_t w = (3 + (uint64_t)L) * k, p = 1;
    for (uint32_t s = 1; s <= L; ++s) { p *= 4; w += p * (k + s); }
    return w;
}

void DevicePolish::reserve(uint64_t bytes, uint64_t max_words, uint64_t windows, uint32_t kk, uint64_t budget, PlRun* run) {
    ctx.make_current();
    k = kk;
    const uint64_t want = std::max<uint64_t>(2 * windows, 64);
    run->table_bytes = want * sizeof(DepthSlot);
    if (want > budget)
        throw std::length_error("polish: the contigs' k-mer table (" + std::to_string(run->table_bytes) + " bytes) does not fit half the free device memory");
    d_bytes.ensure(std::max<uint64_t>(bytes, 1)); d_code.ensure(max_words * 8); d_valid.ensure(max_words * 4); d_wcid.ensure(max_words * 4);
    d_mask.ensure(max_words * 4); d_table.ensure(want * sizeof(DepthSlot));
}

void DevicePolish::fill(DeviceSpectrum& spec, DepthSlot* table, uint64_t n_slots, PlRun* run) {
    AcStream* st = &ctx.stream;
    spec.sweep([&](const GsSlot* spec_table, uint64_t spec_slots, uint64_t parts, uint64_t part) {
        AcTimer timer(st);
        ac_launch("pl_fill", st, PlFillBody{table, spec_table, spec_slots, parts, part}, n_slots);
        timer.stop();
        ac_sync(st);
        run->fill_ms += timer.ms();
    }, &run->sweep);
}

void DevicePolish::pack(const uint8_t* bytes, const uint64_t* len, uint32_t n, uint64_t windows, PlRun* run) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    std::vector<DpContig> contig(n + 1);
    uint64_t off = 0;
    words = 0;
    for (uint32_t c = 0; c < n; ++c) {
        contig[c] = DpContig{off, len[c], words};
        off += len[c]; words += len[c] / 32 + 1;
    }
    contig[n] = DpContig{off, 0, words};
    slots = std::max<uint64_t>(2 * windows, 64);
    if (off > d_bytes.cap || words * 8 > d_code.cap || slots * sizeof(DepthSlot) > d_table.cap)
        throw std::logic_error("polish: a round outgrew the buffers reserved for it");
    d_contig.ensure((n + 1) * sizeof(DpContig));
    if (off) ac_h2d(d_bytes.p, bytes, off, st);
    ac_h2d(d_contig.p, contig.data(), (n + 1) * sizeof(DpContig), st);
    ac_memset(d_table.p, 0, slots * sizeof(DepthSlot), st);
    AcTimer tp(st);
    ac_launch("pl_pack", st, DpPackBody{d_bytes.as<uint8_t>(), d_contig.as<DpContig>(), n, d_code.as<uint64_t>(), d_valid.as<uint32_t>(),
                                        d_wcid.as<uint32_t>()}, words);
    ac_launch("pl_claim", st, QvClaimBody{d_code.as<uint64_t>(), d_valid.as<uint32_t>(), k, d_table.as<DepthSlot>(), slots}, words);
    tp.stop();
    ac_sync(st);
    run->pack_ms += tp.ms();
}

void DevicePolish::windows(DeviceSpectrum& spec, const uint8_t* bytes, const uint64_t* len, uint32_t n, uint64_t windows, uint32_t t,
                           uint32_t* mask, PlRun* run) {
    pack(bytes, len, n, windows, run);
    AcStream* st = &ctx.stream;
    fill(spec, d_table.as<DepthSlot>(), slots, run);
    AcTimer ts(st);
    ac_launch("pl_support", st, PlSupportBody{d_code.as<uint64_t>(), d_valid.as<uint32_t>(), k, d_table.as<DepthSlot>(), slots, t,
                                              d_mask.as<uint32_t>()}, words);
    ts.stop();
    if (words) ac_d2h(mask, d_mask.p, words * 4, st);
    ac_sync(st);
    run->fill_ms += ts.ms();
}

void DevicePolish::score(DeviceSpectrum& spec, const PlLocus* loci, uint64_t n, uint32_t L, uint32_t t, uint64_t budget,
                         const std::function<void(uint64_t, uint64_t, const uint32_t*)>& each, PlRun* run) {
    if (!n) return;
    ctx.make_current();
    AcStream* st = &ctx.stream;
    const uint64_t C = candidates(L), cw = candidate_windows(k, L), per = budget / (2 * cw);
    if (!per)
        throw std::length_error("polish: one locus's candidate table (" + std::to_string(2 * cw * sizeof(DepthSlot)) +
                                " bytes) does not fit the free device memory");
    const uint64_t batch = std::min(n, per);
    d_loci.ensure(batch * sizeof(PlLocus)); d_score.ensure(batch * C * 4); d_out.ensure(batch * 12);
    d_cand.ensure(std::max<uint64_t>(2 * batch * cw, 64) * sizeof(DepthSlot));
    for (uint64_t b0 = 0; b0 < n; b0 += batch) {
        const uint64_t nb = std::min(batch, n - b0), cslots = std::max<uint64_t>(2 * nb * cw, 64);
        DepthSlot* cand = d_cand.as<DepthSlot>();
        run->candidate_bytes = std::max<uint64_t>(run->candidate_bytes, cslots * sizeof(DepthSlot));
        ++run->batches;
        ac_h2d(d_loci.p, loci + b0, nb * sizeof(PlLocus), st);
        ac_memset(cand, 0, cslots * sizeof(DepthSlot), st);
        AcTimer tc(st);
        ac_launch("pl_candidate", st, PlCandidateBody{d_code.as<uint64_t>(), d_valid.as<uint32_t>(), d_loci.as<PlLocus>(), k, L, (uint32_t)C,
                                                      cand, cslots}, nb * C);
        tc.stop();
        ac_sync(st);
        run->candidate_ms += tc.ms();
        fill(spec, cand, cslots, run);
        AcTimer ts(st);
        ac_launch("pl_score", st, PlScoreBody{d_code.as<uint64_t>(), d_valid.as<uint32_t>(), d_loci.as<PlLocus>(), k, L, (uint32_t)C, cand,
                                              cslots, t, d_score.as<uint32_t>()}, nb * C);
        ts.stop();
        each(b0, nb, d_score.as<uint32_t>());                // synchronizes the stream
        run->candidate_ms += ts.ms();
    }
}

void DevicePolish::choose(DeviceSpectrum& spec, const PlLocus* loci, uint64_t n, uint32_t L, uint32_t t, uint64_t budget, uint32_t* out,
                          PlRun* run) {
    AcStream* st = &ctx.stream;
    const uint32_t C = (uint32_t)candidates(L);
    score(spec, loci, n, L, t, budget, [&](uint64_t b0, uint64_t nb, const uint32_t* score) {
        AcTimer tx(st);
        ac_launch("pl_choose", st, PlChooseBody{score, C, d_out.as<uint32_t>()}, nb * 32);
        tx.stop();
        ac_d2h(out + 3 * b0, d_out.p, nb * 12, st);
        ac_sync(st);
        run->choose_ms += tx.ms();
    }, run);
}
