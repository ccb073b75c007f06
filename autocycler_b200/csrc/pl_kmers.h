// The candidate-edit side of the packed k-mer stream, shared by `polish` (polish.cu) and `variants` (variants.cu): a query table's read
// counts filled from a spectrum partition, a candidate edit's checked windows rolled from the packed codes, their claim in a candidate
// table and their score (DESIGN.md §22, §23).
// Device code only.  The bodies sit in an anonymous namespace on purpose: each file that includes this header launches its own kernels
// of them, as polish.cu did when they were its own.
#pragma once
#include "commands.h"
#include "dp_kmers.h"

namespace {
// One thread per slot of a query table, for the keys of spectrum partition `part`: the key's read count r.
struct PlFillBody {
    DepthSlot* table; const GsSlot* spec; uint64_t spec_slots, parts, part;
    AC_D void operator()(uint64_t s) const {
        const uint64_t tag = table[s].key;
        if (!tag) return;
        const uint64_t h = gs_mix(tag - 1);
        if (ac_umul64hi(h, parts) == part) table[s].count = ua_read_count(spec, spec_slots, parts, h, tag - 1);
    }
};

// Calls f(canonical key) for each checked window of candidate c at locus lo, in order: the windows of the edited sequence that start
// at a, k + s of them, rolled over the round's bases [a, p0), the edit's bases and the round's bases from p0 + skip to the span's end
// p0 + d + k.  False (possibly after some calls) when the candidate is not allowed, a deletion past the contig's last base or, on a linear
// contig, a window past its end, or when a checked base is not A/C/G/T.
template <class F> AC_D bool pl_each_key(const uint64_t* code, const uint32_t* valid, const PlLocus& lo, uint32_t c, uint32_t k, uint32_t L,
                                         F&& f) {
    const uint64_t n = lo.len, p0 = lo.a + k - 1 < n ? lo.a + k - 1 : lo.a + k - 1 - n;
    uint32_t b = 0;
    auto base = [&](uint64_t i) {                            // the round's base at i (cyclic on a circular contig); false: not A/C/G/T
        if (i >= n) i -= n;
        const uint64_t w = lo.word0 + i / 32;
        const uint32_t o = (uint32_t)(i % 32);
        b = (uint32_t)(code[w] >> (2 * o)) & 3u;
        return ((valid[w] >> o) & 1u) != 0;
    };
    base(p0);
    const PlEdit e = pl_edit(c, L, b);
    const uint64_t d = e.mlen ? 0 : e.skip;
    if (p0 + d > n || (!lo.circular && p0 + d + k > n)) return false;
    const uint32_t len = 2 * k - 1 + e.mlen + (uint32_t)d - e.skip, top = 2 * (k - 1);
    const uint64_t mask = (1ull << (2 * k)) - 1;
    uint64_t fw = 0, rc = 0;
    for (uint32_t x = 0; x < len; ++x) {
        if (x < k - 1) { if (!base(lo.a + x)) return false; }
        else if (x < k - 1 + e.mlen) b = (e.mid >> (2 * (x - (k - 1)))) & 3u;
        else if (!base(p0 + e.skip + (x - (k - 1) - e.mlen))) return false;
        fw = ((fw << 2) | b) & mask; rc = (rc >> 2) | ((uint64_t)(3 - b) << top);
        if (x >= k - 1) f(fw < rc ? fw : rc);
    }
    return true;
}

// One thread per (locus, candidate): the candidate's checked windows claimed in the candidate table.
struct PlCandidateBody {
    const uint64_t* code; const uint32_t* valid; const PlLocus* loci; uint32_t k, L, C; DepthSlot* table; uint64_t slots;
    AC_D void operator()(uint64_t i) const {
        pl_each_key(code, valid, loci[i / C], (uint32_t)(i % C), k, L, [&](uint64_t key) { dp_claim(table, slots, key); });
    }
};
// One thread per (locus, candidate), after the fill: score[i] = the minimum r over its checked windows when it passes (every window
// allowed, of A/C/G/T bases and with r >= t), else 0.
struct PlScoreBody {
    const uint64_t* code; const uint32_t* valid; const PlLocus* loci; uint32_t k, L, C; const DepthSlot* table; uint64_t slots; uint32_t t;
    uint32_t* score;
    AC_D void operator()(uint64_t i) const {
        uint32_t m = 0xFFFFFFFFu;
        const bool ok = pl_each_key(code, valid, loci[i / C], (uint32_t)(i % C), k, L, [&](uint64_t key) {
            const uint32_t r = qv_read_count(table, slots, key);
            m = r < m ? r : m;
        });
        score[i] = ok && m >= t ? m : 0;
    }
};
}  // namespace
