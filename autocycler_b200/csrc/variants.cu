// Device part of `autocycler variants`: the input's query table filled and every window screened for its three other last bases in one
// sweep over the read spectrum's partitions, the candidates that survive scored by polish's claim, fill and score (DevicePolish::score),
// and each passing candidate's ref count and PK.  Not in the reference (DESIGN.md §23).  This file compiles with nvcc for sm_90a (product)
// and with g++ -DAC_EMULATE (tests/emu, serial execution of the same bodies).
#include "commands.h"
#include "dp_kmers.h"
#include "pl_kmers.h"

#include <algorithm>
#include <vector>

// ------------------------------------------------------------------------------------------------
// variants: fill and screen in one sweep, candidate scores per batch, then ref and PK per passing candidate, see DESIGN.md §23
// ------------------------------------------------------------------------------------------------
namespace {
// One thread per packed word of the input, for the keys of spectrum partition `part`: each window that ends in the word is rolled as
// dp_each_key rolls it, and for each of the three other last bases e the forward and reverse keys get e (two masked ORs, no re-roll).
// Bit i of mask[3 w + j] is set (OR-ed across partitions: each key belongs to one) when that window, with the j-th other base of A, C, G,
// T last, has r >= t.
struct VaScreenBody {
    const uint64_t* code; const uint32_t* valid; uint32_t k; const GsSlot* spec; uint64_t spec_slots, parts, part; uint32_t t; uint32_t* mask;
    AC_D void operator()(uint64_t w) const {
        const uint32_t ends = gs_window_ends(valid[w], w ? valid[w - 1] : 0, k);
        if (!ends) return;
        const uint64_t c = code[w], pc = w ? code[w - 1] : 0, kmask = (1ull << (2 * k)) - 1;
        const uint32_t top = 2 * (k - 1);
        uint64_t fw = 0, rc = 0;
        for (uint32_t i = 32 - (k - 1); i < 32; ++i) {
            const uint64_t b = (pc >> (2 * i)) & 3;
            fw = ((fw << 2) | b) & kmask; rc = (rc >> 2) | ((3 - b) << top);
        }
        uint32_t m0 = 0, m1 = 0, m2 = 0;
        for (uint32_t i = 0; i < 32; ++i) {
            const uint64_t b = (c >> (2 * i)) & 3;
            fw = ((fw << 2) | b) & kmask; rc = (rc >> 2) | ((3 - b) << top);
            if (!((ends >> i) & 1)) continue;
            for (uint32_t j = 0; j < 3; ++j) {
                const uint64_t e = j < b ? j : j + 1;
                const uint64_t f = (fw & ~3ull) | e, r = (rc & ~(3ull << top)) | ((3 - e) << top), key = f < r ? f : r, h = gs_mix(key);
                if (ac_umul64hi(h, parts) != part || ua_read_count(spec, spec_slots, parts, h, key) < t) continue;
                if (j == 0) m0 |= 1u << i;
                else if (j == 1) m1 |= 1u << i;
                else m2 |= 1u << i;
            }
        }
        mask[3 * w] |= m0; mask[3 * w + 1] |= m1; mask[3 * w + 2] |= m2;
    }
};
// One thread per passing candidate: out[2 i] = ref, the least r over the input's windows that start at a .. p + d (cyclic on a circular
// contig; a window with a base that is not A/C/G/T counts 0), out[2 i + 1] = PK, the candidate's checked windows whose key the query
// table holds (an indel's last one, the input's window at p + d, left out).
struct VaRefBody {
    const uint64_t* code; const uint32_t* valid; const VaCandidate* cand; uint32_t k, L; const DepthSlot* table; uint64_t slots; uint32_t* out;
    AC_D void operator()(uint64_t i) const {
        const PlLocus lo = cand[i].lo;
        const uint32_t c = cand[i].c;
        uint32_t pk = 0, last = 0;
        pl_each_key(code, valid, lo, c, k, L, [&](uint64_t key) { last = dp_holds(table, slots, key) ? 1u : 0u; pk += last; });
        if (c >= 3) pk -= last;
        const uint64_t n = lo.len, p0 = lo.a + k - 1 < n ? lo.a + k - 1 : lo.a + k - 1 - n;
        const uint32_t cur = (uint32_t)(code[lo.word0 + p0 / 32] >> (2 * (p0 % 32))) & 3u;
        const PlEdit e = pl_edit(c, L, cur);
        const uint32_t len = 2 * k - 1 + (e.mlen ? 0 : e.skip), top = 2 * (k - 1);
        const uint64_t mask = (1ull << (2 * k)) - 1;
        uint64_t fw = 0, rc = 0;
        uint32_t m = 0xFFFFFFFFu, run = 0;
        for (uint32_t x = 0; x < len; ++x) {
            uint64_t j = lo.a + x;
            if (j >= n) j -= n;
            const uint64_t w = lo.word0 + j / 32;
            const uint32_t o = (uint32_t)(j % 32);
            const uint64_t b = (code[w] >> (2 * o)) & 3;
            run = (valid[w] >> o) & 1u ? run + 1 : 0;
            fw = ((fw << 2) | b) & mask; rc = (rc >> 2) | ((3 - b) << top);
            if (x < k - 1) continue;
            const uint32_t r = run >= k ? qv_read_count(table, slots, fw < rc ? fw : rc) : 0;
            m = r < m ? r : m;
        }
        out[2 * i] = m; out[2 * i + 1] = pk;
    }
};
}  // namespace

void DeviceVariants::screen(DeviceSpectrum& spec, DevicePolish& pl, uint32_t t, uint32_t* mask, PlRun* prun, VaRun* run) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    const uint64_t words = pl.packed_words();
    d_mask.ensure(std::max<uint64_t>(words * 12, 12));
    ac_memset(d_mask.p, 0, words * 12, st);
    spec.sweep([&](const GsSlot* spec_table, uint64_t spec_slots, uint64_t parts, uint64_t part) {
        AcTimer tf(st);
        ac_launch("va_fill", st, PlFillBody{pl.query_table(), spec_table, spec_slots, parts, part}, pl.query_slots());
        tf.stop();
        AcTimer ts(st);
        ac_launch("va_screen", st, VaScreenBody{pl.packed_codes(), pl.packed_valid(), pl.kmer(), spec_table, spec_slots, parts, part, t,
                                                d_mask.as<uint32_t>()}, words);
        ts.stop();
        ac_sync(st);
        prun->fill_ms += tf.ms(); run->screen_ms += ts.ms();
    }, &prun->sweep);
    if (words) ac_d2h(mask, d_mask.p, words * 12, st);
    ac_sync(st);
}

void DeviceVariants::scores(DeviceSpectrum& spec, DevicePolish& pl, const PlLocus* loci, uint64_t n, uint32_t L, uint32_t t, uint64_t budget,
                            uint32_t* score, PlRun* prun) {
    AcStream* st = &ctx.stream;
    const uint64_t C = DevicePolish::candidates(L);
    pl.score(spec, loci, n, L, t, budget, [&](uint64_t b0, uint64_t nb, const uint32_t* d_score) {
        ac_d2h(score + b0 * C, d_score, nb * C * 4, st);
        ac_sync(st);
    }, prun);
}

void DeviceVariants::ref(DevicePolish& pl, const VaCandidate* cand, uint64_t n, uint32_t L, uint32_t* out, VaRun* run) {
    if (!n) return;
    ctx.make_current();
    AcStream* st = &ctx.stream;
    d_cand.ensure(n * sizeof(VaCandidate)); d_out.ensure(n * 8);
    ac_h2d(d_cand.p, cand, n * sizeof(VaCandidate), st);
    AcTimer tr(st);
    ac_launch("va_ref", st, VaRefBody{pl.packed_codes(), pl.packed_valid(), d_cand.as<VaCandidate>(), pl.kmer(), L, pl.query_table(),
                                      pl.query_slots(), d_out.as<uint32_t>()}, n);
    tr.stop();
    ac_d2h(out, d_out.p, n * 8, st);
    ac_sync(st);
    run->ref_ms += tr.ms();
}
