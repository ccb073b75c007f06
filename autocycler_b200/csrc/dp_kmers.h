// The assembly side of the packed k-mer stream, shared by `depth` (depth.cu), `qv` (qv.cu), `unassembled` (unassembled.cu) and `polish`
// (polish.cu): contigs packed like the reads, each from a fresh word that keeps its contig id, the canonical keys of the windows that end
// in a word, the claim of an assembly's keys and the read probe into a DepthSlot table, its lookups, a key's count in a spectrum
// partition's table, and the warp-grouped add (DESIGN.md §19-§22).
// Device code only.  The bodies sit in an anonymous namespace on purpose: each
// file that includes this header launches its own kernels of them, as depth.cu did when they were its own.
#pragma once
#include "commands.h"
#include "gs_kmers.h"

namespace {
struct DpContig { uint64_t off, len, woff; };      // bytes at off, len of them (junction bases included), first packed word

// Adds 1 to *p.  On the device the lanes of a warp that add to the same address are grouped first, one atomic per group: in the
// median's passes every unique key of a long contig adds to the same few bins.
#ifdef AC_EMULATE
inline void dp_add_one(uint32_t* p) { ++*p; }
#else
__device__ __forceinline__ void dp_add_one(uint32_t* p) {
    const unsigned same = __match_any_sync(__activemask(), (unsigned long long)p);
    if ((int)(threadIdx.x & 31) == __ffs((int)same) - 1) atomicAdd(p, (unsigned)__popc(same));
}
#endif

// Calls f(canonical key) for each window that ends in word w: the forward and reverse keys roll over word w-1's last k-1 bases and then
// w's 32, as GsCountBody's do.
template <class F> AC_D void dp_each_key(const uint64_t* code, const uint32_t* valid, uint64_t w, uint32_t k, F&& f) {
    const uint32_t ends = gs_window_ends(valid[w], w ? valid[w - 1] : 0, k);
    if (!ends) return;
    const uint64_t c = code[w], pc = w ? code[w - 1] : 0, mask = (1ull << (2 * k)) - 1;
    const uint32_t top = 2 * (k - 1);
    uint64_t fw = 0, rc = 0;
    for (uint32_t i = 32 - (k - 1); i < 32; ++i) {
        const uint64_t b = (pc >> (2 * i)) & 3;
        fw = ((fw << 2) | b) & mask; rc = (rc >> 2) | ((3 - b) << top);
    }
    for (uint32_t i = 0; i < 32; ++i) {
        const uint64_t b = (c >> (2 * i)) & 3;
        fw = ((fw << 2) | b) & mask; rc = (rc >> 2) | ((3 - b) << top);
        if ((ends >> i) & 1) f(fw < rc ? fw : rc);
    }
}

// One thread per packed word of the assembly: its contig (a binary search over the word offsets), codes, validity mask and contig id.
struct DpPackBody {
    const uint8_t* bytes; const DpContig* contig; uint32_t n; uint64_t* code; uint32_t* valid; uint32_t* wcid;
    AC_D void operator()(uint64_t w) const {
        uint32_t lo = 0, hi = n;                             // the last contig whose first word is <= w
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) / 2; if (contig[mid].woff <= w) lo = mid; else hi = mid; }
        const DpContig o = contig[lo];
        uint64_t c;
        valid[w] = gs_pack_word(bytes + o.off, o.len, w - o.woff, &c);
        code[w] = c;
        wcid[w] = lo;
    }
};
// One thread per packed word of the reads: each window is a lookup that stops at its key or the first empty slot.  A hit on a unique
// key adds 1 while a plain read shows the count below 2^31 (GsCountBody's guard).
struct DpProbeBody {
    const uint64_t* code; const uint32_t* valid; uint32_t k; DepthSlot* table; uint64_t slots;
    AC_D void operator()(uint64_t w) const {
        dp_each_key(code, valid, w, k, [&](uint64_t key) {
            uint64_t s = ac_umul64hi(gs_mix(key), slots);
            const uint64_t tag = key + 1;
            for (;;) {
                DepthSlot* q = table + s;
                const uint64_t cur = q->key;
                if (cur == 0) return;
                if (cur == tag) {
                    if (!(q->flags & AC_DEPTH_DUP) && ac_ld_volatile(&q->count) < 0x80000000u) ac_atomic_add(&q->count, 1u);
                    return;
                }
                if (++s == slots) s = 0;
            }
        });
    }
};
// Claims a key in a DepthSlot table by linear probing from its home slot with a CAS on the empty key.
AC_D void dp_claim(DepthSlot* table, uint64_t slots, uint64_t key) {
    uint64_t s = ac_umul64hi(gs_mix(key), slots);
    const uint64_t tag = key + 1;
    for (;;) {
        DepthSlot* q = table + s;
        uint64_t cur = ac_ld_volatile(&q->key);
        if (cur == 0) cur = ac_atomic_cas(&q->key, (uint64_t)0, tag);
        if (cur == 0 || cur == tag) return;
        if (++s == slots) s = 0;
    }
}
// One thread per packed word of every assembly: each window's key is claimed (dp_claim); the flags stay 0, so DpProbeBody counts every
// read window that hits the key.
struct QvClaimBody {
    const uint64_t* code; const uint32_t* valid; uint32_t k; DepthSlot* table; uint64_t slots;
    AC_D void operator()(uint64_t w) const {
        dp_each_key(code, valid, w, k, [&](uint64_t key) { dp_claim(table, slots, key); });
    }
};
// The reads' count of a key the combined table holds.
AC_D uint32_t qv_read_count(const DepthSlot* table, uint64_t slots, uint64_t key) {
    uint64_t s = ac_umul64hi(gs_mix(key), slots);
    for (;;) {
        const DepthSlot* q = table + s;
        if (q->key == key + 1) return q->count;
        if (q->key == 0) return 0;
        if (++s == slots) s = 0;
    }
}
// The read count of a key of partition `part` of the read spectrum (h: its mix) in that partition's table, which holds every such key.
AC_D uint32_t ua_read_count(const GsSlot* table, uint64_t slots, uint64_t parts, uint64_t h, uint64_t key) {
    uint64_t s = ac_umul64hi(h * parts, slots);
    for (;;) {
        const GsSlot q = table[s];
        if (q.key == key + 1) return q.count;
        if (q.key == 0) return 0;
        if (++s == slots) s = 0;
    }
}
// Whether the claimed table holds a key.
AC_D bool dp_holds(const DepthSlot* table, uint64_t slots, uint64_t key) {
    uint64_t s = ac_umul64hi(gs_mix(key), slots);
    for (;;) {
        const uint64_t cur = table[s].key;
        if (cur == key + 1) return true;
        if (cur == 0) return false;
        if (++s == slots) s = 0;
    }
}
}  // namespace
