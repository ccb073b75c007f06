// Device pipeline: k-mer table build, adjacency, unitig occurrences ("runs"), unitig identity,
// seed k-mers and links.  Every kernel is a functor body (backend.h); this file compiles with nvcc
// for sm_90a (product) and with g++ -DAC_EMULATE (tests/emu, serial host execution of the same bodies).
//
// Order-free restatement of the reference's serial walk (unitig_graph.rs:176-226), see DESIGN.md §3:
//   * per canonical k-mer: depth, first/last flags, node-centric in/out degree over ". A C G T"
//   * an edge K->K' is merged iff outdeg(K)==1, !last(K), indeg(K')==1, !first(K'), K' != K, K' != rc(K)
//   * unitigs are the maximal chains of merged edges; because every occurrence of a chain member is
//     preceded/followed by its chain neighbours, the chains are exactly the maximal runs of merged
//     edges ALONG THE INPUT SEQUENCES, so chain construction is a flag + scan over positions instead
//     of list ranking over a hash table.
#include "pipeline.h"

#include <algorithm>
#include <cmath>
#include <vector>

unsigned long long g_ac_kernel_launches = 0;

#define AC_NONE32 0xFFFFFFFFu
#define AC_CHUNK 32            // windows per thread in the insert kernel
#define AC_MINCHUNK 128        // windows per thread in the seed-k-mer kernel
#define AC_MAX_RANKS 16         // ranks of one multi-GPU build (one box)
#define AC_BOUND_STRIPES 64     // power of two: accumulators that every candidate adds to are striped
// Resident 256-thread CTAs per SM the insert kernel is compiled for, i.e. its register budget (65536 / (256 x CTAS) registers per
// thread).  profiles/insert_budget_sweep.py builds the library at other values and times the insert; DESIGN.md §4 has the numbers.
#ifndef AC_INSERT_CTAS
#define AC_INSERT_CTAS 2
#endif

// ------------------------------------------------------------------------------------------------
// small device helpers
// ------------------------------------------------------------------------------------------------
struct TableView {
    Slot* slots;
    uint64_t cap;
    const uint64_t* packed;
    const SeqInfo* seqs;
    uint32_t n_seqs;
    uint32_t* count_big;        // null, or (after a 20-bit count neared its end) the depth of every slot in 32 bits; the slots' own count fields then stay 0
    uint32_t gb;                // bits of a slot's occurrence pointer (slot_gpos_bits(total)); the fingerprint gets the rest
    uint32_t alarm;             // a loaded slot count of this much or more raises the count alarm (AC_SLOT_COUNT_ALARM; tests lower it)
};
// Linear probing starts at the first slot of a 32-byte group of four (cap is a multiple of 4): one sector holds the whole first probe.
AC_D uint64_t table_home(const TableView& t, uint64_t h) { return ac_umul64hi(h, t.cap >> 2) << 2; }
AC_D uint32_t table_depth(const TableView& t, uint64_t slot) { return t.count_big ? t.count_big[slot] : slot_count(t.slots[slot]); }

template <int W> AC_D Key<W> window_key(const TableView& t, uint64_t g, bool dotted, const KParams& p) {
    Key<W> key = fetch_codes<W>(t.packed, g, p);
    if (dotted) {
        const SeqInfo s = t.seqs[find_seq(t.seqs, t.n_seqs, g)];
        key.d = window_dots(s, g - s.start, p.k);
    }
    return key;
}

// Find the slot holding k-mer `a` (whose reverse complement is `arc`), or AC_NONE32.
template <int W> AC_D uint32_t table_find(const TableView& t, const Key<W>& a, const Key<W>& arc, const KParams& p) {
    const uint64_t h = key_hash(key_select(key_is_canonical(a, p), a, arc));
    const uint32_t tag = make_tag(a.d != 0, h, t.gb);
    uint64_t slot = table_home(t, h);
    for (;;) {
        const Slot e = t.slots[slot];
        if (e == AC_EMPTY_SLOT) return AC_NONE32;
        if (slot_tag(e, t.gb) == tag) {
            Key<W> rep = window_key<W>(t, slot_gpos(e, t.gb), a.d != 0, p);
            if (key_eq(rep, a) || key_eq(rep, arc)) return (uint32_t)slot;
        }
        if (++slot == t.cap) slot = 0;
    }
}

// An occurrence (or, in the multi-GPU merge, another rank's `add` occurrences) of the k-mer that slot `slot` already holds: the
// count goes up, missing flags are set, and with `track_min` the slot ends up pointing at the smallest occurrence (a name for the
// k-mer that does not depend on the rank).  `seen` is the slot word the caller compared against.  counters[2] is the probe-limit
// flag, counters[3] the count alarm.
AC_D void slot_add_occurrence(const TableView& t, uint64_t slot, Slot seen, uint64_t g, uint32_t add, uint32_t flags, bool track_min, unsigned long long* counters) {
    if (!t.count_big && slot_count(seen) + add >= t.alarm) counters[3] = 1;       // from the copy the caller loaded: see the slot layout in kmer_key.h
    if (!track_min) {
        if (t.count_big) ac_atomic_add(&t.count_big[slot], add);
        else ac_atomic_add(&t.slots[slot], (uint64_t)add << AC_SLOT_COUNT_SHIFT);            // result unused: a fire-and-forget reduction, nobody waits for the old value
        if (flags & ~slot_flags(seen)) ac_atomic_or(&t.slots[slot], (uint64_t)flags);     // usually there already (`seen` may be stale: then the OR is merely redundant)
        return;
    }
    if (t.count_big) ac_atomic_add(&t.count_big[slot], add);
    Slot old = seen;
    for (;;) {
        Slot nw = old | flags;
        if (!t.count_big) { nw += (uint64_t)add << AC_SLOT_COUNT_SHIFT; if (slot_count(old) + add >= t.alarm) counters[3] = 1; }
        if (g < slot_gpos(old, t.gb)) nw = slot_with_gpos(nw, g, t.gb);
        const Slot was = ac_atomic_cas(&t.slots[slot], old, nw);
        if (was == old) return;
        old = was;
    }
}

// Calls f(succ, succ_rc) for every k-mer that could follow `a` (kmer_graph.rs:136-150): drop the first
// symbol, append one of ". A C G T".  Combinations that would put a base after a dot, or dots on both
// ends (impossible because every contig has L >= k), cannot exist in the graph and are skipped.
template <int W, class F> AC_D void for_each_successor(const Key<W>& a, const Key<W>& arc, bool any_dotted, const KParams& p, F&& f) {
    if (a.d == 0) {
        for (uint64_t x = 0; x < 4; ++x) {
            Key<W> s = a, src = arc;
            key_push_right(s, x, p); key_push_left(src, 3 - x, p);
            f(s, src);
        }
        if (any_dotted) { Key<W> s = a; key_push_right(s, 0, p); s.d = -1; f(s, key_rc(s, p)); }
    } else if (a.d > 0) {               // p leading dots -> p-1 leading dots, any base appended
        for (uint64_t x = 0; x < 4; ++x) { Key<W> s = a; key_push_right(s, x, p); s.d = a.d - 1; f(s, key_rc(s, p)); }
        if (a.d == 1) { Key<W> s = a; key_push_right(s, 0, p); s.d = -1; f(s, key_rc(s, p)); }   // ".X" -> "X." (k-1 bases then a dot)
    } else {                            // trailing dots: only another dot can follow
        Key<W> s = a; key_push_right(s, 0, p); s.d = a.d - 1; f(s, key_rc(s, p));
    }
}

// ------------------------------------------------------------------------------------------------
// kernel bodies
// ------------------------------------------------------------------------------------------------
// ASCII -> 2-bit packed, 32 bases per thread ('.' -> 0; the dot runs are described by SeqInfo).  The same thread decides whether the 32
// windows that START in its word form an interior block: all of them, the window before and the window after are windows of one
// sequence, free of dots, none first or last (one byte per block; the insert kernel reads it instead of searching the sequence table).
struct PackBody {
    const uint8_t* ascii; uint64_t total; uint64_t* packed; const SeqInfo* seqs; uint32_t n_seqs; uint8_t* interior;
    AC_D void operator()(uint64_t i) const {
        uint64_t word = 0;
        const uint64_t base = i * 32;
        for (uint32_t j = 0; j < 32; ++j) {
            const uint64_t g = base + j;
            const uint64_t code = g < total ? base_code(ascii[g]) : 0;
            word |= code << (62 - 2 * j);
        }
        packed[i] = word;
        if (interior) {
            const SeqInfo s = seqs[find_seq(seqs, n_seqs, base)];
            const uint64_t fs0 = base - s.start;
            interior[i] = fs0 >= (uint64_t)s.lead + 1 && fs0 + 33 + s.trail <= s.len ? 1 : 0;
        }
    }
};

// kmer_graph.rs:92-134 add_sequence, both strands at once: one canonical entry per k-mer, count = depth.
// A warp takes the 64 windows that start in two consecutive 32-base words of the packed store (units are aligned to 64 coordinates),
// and lane l owns two of them, g0 + l and g0 + 32 + l: the W+3 packed words both keys, their left and their right neighbour bases are
// cut from sit at the same addresses for all of its lanes (one transaction each), and the slot-id stores coalesce (one 128-byte store
// per half).  Almost every 32-window half lies in the interior of one sequence: no dots, no first or last window, every window has
// both neighbours — that case is decided once per half and skips the per-window bookkeeping.  The table is probed a 32-byte group of
// four slots at a time (one sector, one 256-bit load; the home slot of a k-mer is the first of a group and the probe order is plain
// linear probing from there), in two phases: a cheap scan to the first slot that is empty (claimed at once, count and flags in the
// same CAS) or carries the k-mer's 6-bit tag, then — lanes together again — the comparison with the occurrence that slot points at.
// Each probe is a chain of dependent loads; a lane runs the chains of its two windows side by side, so that twice as many loads are in
// flight per warp (DESIGN.md §4).
template <int W> struct InsertBody {
    TableView t; KParams p;
    const uint8_t* interior;            // [total / 32] PackBody's flag per block of 32 coordinates
    uint32_t g_first;                   // coordinate of unit 0, a multiple of 64 (inputs are limited to 2^32 - 2 padded bytes: coordinates fit 32 bits)
    uint32_t g_begin, g_end;            // coordinates of the sequences this rank owns
    bool track_min;                     // multi-GPU: the slot must end up pointing at the SMALLEST occurrence
    uint32_t* pos_slot;                 // [total] slot of the window starting at each global coordinate (null in the sizing pass)
    unsigned long long* counters;       // [0] slots claimed (sizing pass only), [1] dotted k-mers claimed, [2] probe-limit flag, [3] count alarm
    bool sizing;                        // the sizing pass: the caller has picked the windows (SampleBody), only distinct k-mers are counted
    uint32_t* claimed_bits;             // [total / 32] bit j of word w: the window at coordinate 32w + j claimed its slot, i.e. it is the first occurrence of a distinct k-mer (the list of distinct k-mers is made from these); null in the sizing pass
    struct Unit { Key<W> fwd, rc; uint64_t h; uint32_t flags, g; bool valid; };
    // window l of an interior block: x = the packed word before the block, then the block's own W+1 words
    AC_D void interior_unit(uint32_t l, const uint64_t (&x)[W + 2], Unit& u) const {
        uint64_t xs[W + 1];
#pragma unroll
        for (int j = 0; j <= W; ++j) xs[j] = x[j + 1];
        const uint32_t sh = 2 * l;
        uint64_t y[W];
        ac_stream_window<W>(xs, sh, y);      // y = the 64W bits of the base stream that start at bit `sh` of the block's first word
        const uint32_t al = 64 - p.top_bits;
#pragma unroll
        for (int j = W - 1; j >= 0; --j) { uint64_t v = y[j] >> al; if (al && j > 0) v |= y[j - 1] << (64 - al); u.fwd.w[j] = v; }
        u.fwd.d = 0;
        u.rc = key_rc(u.fwd, p);
        const bool canon_fwd = key_is_canonical(u.fwd, p);
        // the base after the window is base k of the stream that starts at the window: 32(W-1) < k < 32W, so it lies in y[W-1]
        const uint32_t nb = (uint32_t)(y[W - 1] >> (62 - 2 * (p.k & 31u))) & 3u;
        const uint32_t pb = l ? (uint32_t)(xs[0] >> (64 - sh)) & 3u : (uint32_t)x[0] & 3u;
        const uint32_t out_b = canon_fwd ? nb : 3u - pb, in_b = canon_fwd ? pb : 3u - nb;
        u.flags = (1u << (AC_AUX_OBS_OUT_SHIFT + out_b)) | (1u << (AC_AUX_OBS_IN_SHIFT + in_b));
        u.h = key_hash(key_select(canon_fwd, u.fwd, u.rc));     // by value: a choice between the two references would keep the units in local memory
        u.valid = true;
    }
    // a window of a block at the end of a sequence, between two sequences or at the edge of the shard; false: no window starts at g
    AC_D bool edge_unit(uint32_t g, Key<W>& fwd, Key<W>& rc, uint64_t& h, uint32_t& flags) const {
        const SeqInfo s = t.seqs[find_seq(t.seqs, t.n_seqs, g)];
        const uint64_t fs = g - s.start;
        if (!(g >= g_begin && g < g_end && fs < s.len)) return false;        // outside the shard, or one of the k-1 padded bytes that start no window
        fwd = fetch_codes<W>(t.packed, g, p);
        fwd.d = window_dots(s, fs, p.k);
        rc = key_rc(fwd, p);
        const bool canon_fwd = key_is_canonical(fwd, p);
        flags = 0;
        // Kmer::first_position (kmer_graph.rs:57-60): position 0 of the forward strand is window 0; position 0 of the
        // reverse strand is the reverse complement of the last window (kmer_graph.rs:103-108).
        if (fs == 0) flags |= canon_fwd ? AC_AUX_FIRST_CANON : AC_AUX_FIRST_RC;
        if (fs + 1 == s.len) flags |= canon_fwd ? AC_AUX_FIRST_RC : AC_AUX_FIRST_CANON;
        if (fwd.d == 0) {    // neighbouring bases seen next to this k-mer: spares the adjacency kernel the probes for neighbours it already knows to exist
            if (fs + 1 < s.len && window_dots(s, fs + 1, p.k) == 0) {
                const uint32_t b = packed_base(t.packed, (uint64_t)g + p.k);
                flags |= canon_fwd ? (1u << (AC_AUX_OBS_OUT_SHIFT + b)) : (1u << (AC_AUX_OBS_IN_SHIFT + 3 - b));
            }
            if (fs > 0 && window_dots(s, fs - 1, p.k) == 0) {
                const uint32_t b = packed_base(t.packed, (uint64_t)g - 1);
                flags |= canon_fwd ? (1u << (AC_AUX_OBS_IN_SHIFT + b)) : (1u << (AC_AUX_OBS_OUT_SHIFT + 3 - b));
            }
        }
        h = key_hash(key_select(canon_fwd, fwd, rc));
        return true;
    }
    // Enters the k-mers of the lane's N windows (or finds them) and counts the occurrences.  All lanes of the warp call this together.
    // The windows are probed side by side: every round loads the next group of each window still scanning before it looks at any of
    // them, and fetches the stored occurrences of all windows that met their tag before it compares any.  `home_group`, when given,
    // is window 0's home group, already in registers.
    template <int N> AC_D void upsert(const Unit (&u)[N], const Slot* home_group = nullptr) const {
        const uint32_t tag_mask = (1u << AC_SLOT_TAG_BITS(t.gb)) - 1u;
        // An empty slot is all ones and no window starts at coordinate 2^gb - 1, so "empty" is a test of the occurrence pointer alone: the
        // high word at or above this value.  The tag sits at bits 30.. of the slot; slot_tag_word() brings it down with one funnel shift.
        const uint32_t empty_hi = 0xFFFFFFFFu << (32u - t.gb);
        bool dotted[N], done[N], failed[N];
        uint32_t tag[N], probes[N], fresh[N];      // fresh: lanes of this warp whose window claimed a slot
        uint64_t slot[N];
#pragma unroll
        for (int w = 0; w < N; ++w) {
            dotted[w] = u[w].valid && u[w].fwd.d != 0;
            tag[w] = make_tag(dotted[w], u[w].h, t.gb);
            slot[w] = table_home(t, u[w].h);
            done[w] = !u[w].valid; failed[w] = false; probes[w] = 0; fresh[w] = 0;
        }
        bool fetched = home_group != nullptr;      // the home group is in registers already: good for the first look at it only
        for (;;) {
            bool claimed[N], scanning[N]; Slot q[N];
#pragma unroll
            for (int w = 0; w < N; ++w) { claimed[w] = false; q[w] = 0; scanning[w] = !done[w]; }
            for (;;) {
                Slot grp[N][4];
#pragma unroll
                for (int w = 0; w < N; ++w) {
                    if (!scanning[w]) continue;
                    if (w == 0 && fetched) { grp[0][0] = home_group[0]; grp[0][1] = home_group[1]; grp[0][2] = home_group[2]; grp[0][3] = home_group[3]; }      // may lag the table, as any load may (see slot_add_occurrence)
                    else ac_ld_group(t.slots + (slot[w] & ~3ull), grp[w]);
                }
                fetched = false;
                bool more = false;
#pragma unroll
                for (int w = 0; w < N; ++w) {
                    if (!scanning[w]) continue;
                    // the first slot of the group, from `slot` on, that is empty or carries the tag
                    const uint64_t base = slot[w] & ~3ull;
                    uint32_t cand = 0;
#pragma unroll
                    for (uint32_t j = 0; j < 4; ++j) {
                        const bool is_empty = (uint32_t)(grp[w][j] >> 32) >= empty_hi;
                        const bool has_tag = ((slot_tag_word(grp[w][j]) ^ tag[w]) & tag_mask) == 0;
                        cand |= (is_empty || has_tag) ? 1u << j : 0u;
                    }
                    cand &= 0xFu << (slot[w] & 3u);
                    if (cand == 0) {
                        slot[w] = base + 4; if (slot[w] >= t.cap) slot[w] = 0;
                        if (++probes[w] > 2048) { counters[2] = 1; failed[w] = true; done[w] = true; scanning[w] = false; }    // the table was sized too small: the host retries with the safe size
                        else more = true;
                        continue;
                    }
                    const uint32_t j = (uint32_t)ac_ctz(cand);
                    slot[w] = base + j;
                    q[w] = j == 0 ? grp[w][0] : j == 1 ? grp[w][1] : j == 2 ? grp[w][2] : grp[w][3];
                    if ((uint32_t)(q[w] >> 32) >= empty_hi) {
                        q[w] = ac_atomic_cas(&t.slots[slot[w]], (Slot)AC_EMPTY_SLOT, make_slot(u[w].g, tag[w], t.count_big ? 0u : 1u, u[w].flags, t.gb));
                        if (q[w] == AC_EMPTY_SLOT) { claimed[w] = true; scanning[w] = false; continue; }
                        if (slot_tag(q[w], t.gb) != tag[w]) { ++slot[w]; if (slot[w] >= t.cap) slot[w] = 0; more = true; continue; }      // somebody else's k-mer got there first: on to the next slot
                    }
                    scanning[w] = false;
                }
                if (!more) break;
            }
#ifdef __CUDA_ARCH__
            __syncwarp();
#pragma unroll
            for (int w = 0; w < N; ++w) fresh[w] |= __ballot_sync(0xFFFFFFFFu, !done[w] && claimed[w]);          // a claimed slot is a new distinct k-mer
#else
            for (int w = 0; w < N; ++w) if (!done[w] && claimed[w]) fresh[w] = 1;
#endif
            Key<W> rep[N] = {};
#pragma unroll
            for (int w = 0; w < N; ++w) if (!done[w] && !claimed[w]) rep[w] = window_key<W>(t, slot_gpos(q[w], t.gb), dotted[w], p);
#pragma unroll
            for (int w = 0; w < N; ++w) {
                if (done[w]) continue;
                if (claimed[w]) {
                    if (t.count_big) ac_atomic_add(&t.count_big[slot[w]], 1u);
                    if (sizing) ac_atomic_add(&counters[0], 1ull);
                    if (dotted[w]) ac_atomic_add(&counters[1], 1ull);
                    done[w] = true;
                } else if (key_eq(rep[w], u[w].fwd) || key_eq(rep[w], u[w].rc)) {
                    if (!sizing) slot_add_occurrence(t, slot[w], q[w], u[w].g, 1u, u[w].flags, track_min, counters);
                    done[w] = true;
                } else if (++slot[w] == t.cap) slot[w] = 0;
            }
            bool all_done = true;
#pragma unroll
            for (int w = 0; w < N; ++w) all_done = all_done && done[w];
#ifdef __CUDA_ARCH__
            if (__all_sync(0xFFFFFFFFu, all_done)) break;
#else
            if (all_done) break;
#endif
        }
#pragma unroll
        for (int w = 0; w < N; ++w) {
            if (u[w].valid && !failed[w] && pos_slot) ac_st_stream(&pos_slot[u[w].g], (uint32_t)slot[w]);
            if (!claimed_bits) continue;
#ifdef __CUDA_ARCH__
            if ((threadIdx.x & 31u) == 0) claimed_bits[u[w].g >> 5] = fresh[w];      // each half's 32 windows start in one word of coordinates
#else
            if (fresh[w]) claimed_bits[u[w].g >> 5] |= 1u << (u[w].g & 31u);
#endif
        }
    }
    AC_D void prepare(uint64_t i, Unit (&u)[2]) const {
        const uint32_t g0 = g_first + (uint32_t)(i >> 5) * 64u, l = (uint32_t)i & 31u, i0 = g0 >> 5;
        bool inner[2];
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            const uint64_t b = (uint64_t)g0 + 32u * s;
            inner[s] = b >= g_begin && b + 32 <= g_end && interior[i0 + s];
        }
        uint64_t x[W + 3] = {};              // the word before the unit, then the W+2 words from the unit's first on
        if (inner[0] || inner[1]) {
            if (inner[0]) x[0] = t.packed[i0 - 1];
#pragma unroll
            for (int j = 0; j <= W + 1; ++j) x[j + 1] = t.packed[i0 + j];
        }
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            u[s].g = g0 + 32u * s + l; u[s].fwd = Key<W>(); u[s].rc = Key<W>(); u[s].h = 0; u[s].flags = 0;
            if (inner[s]) {
                uint64_t xs[W + 2];
#pragma unroll
                for (int j = 0; j <= W + 1; ++j) xs[j] = x[s + j];
                interior_unit(l, xs, u[s]);
            } else u[s].valid = edge_unit(u[s].g, u[s].fwd, u[s].rc, u[s].h, u[s].flags);
        }
    }
    AC_D void operator()(uint64_t i) const {
        Unit u[2]; prepare(i, u);
#ifdef AC_EMULATE
        Slot grp[4] = {0, 0, 0, 0};          // the CPU suite also takes the route with window 0's home group handed in by the caller
        if (u[0].valid && !sizing) { ac_ld_group(t.slots + table_home(t, u[0].h), grp); upsert<2>(u, grp); return; }
#endif
        upsert<2>(u);
    }
};

// The sizing pass: how many distinct canonical k-mers are there?  A k-mer is sampled when a hash of the seven bases around its centre,
// read on its canonical strand, ends in six zero bits — a property of the k-mer, so it is kept or dropped with ALL its occurrences and
// 64 x the number of distinct sampled k-mers estimates the total.  The test costs a few instructions per window (the centre bases roll
// along the packed words); only the ~1/64 of the windows that pass build their keys and enter the small sample table.  Windows with
// dots (at most k-1 per sequence end) are left out: they cannot move the estimate.  One thread scans 32 consecutive windows.
template <int W> struct SampleBody {
    InsertBody<W> ins; uint32_t total;
    AC_D static bool sampled(uint32_t centre7) {          // centre7: 14 bits, the 7 bases around the centre base, first base most significant
        uint32_t c = centre7;
        if ((c >> 6) & 2u) {                               // centre base G or T: read the other strand (reverse the 7 bases, complement them)
            uint32_t r = 0;
            for (int b = 0; b < 7; ++b) r |= ((c >> (2 * b)) & 3u) << (2 * (6 - b));
            c = ~r & 0x3FFFu;
        }
        return ((c * 0x9E3779B1u) >> 26) == 0;
    }
    AC_D void operator()(uint64_t i) const {
        const uint32_t g0 = (uint32_t)i * 32u;
        const uint32_t k = ins.p.k, h = ins.p.h;
        const bool interior = g0 + 32 <= total && ins.interior[g0 >> 5];
        uint32_t hits = 0;
        if (interior) {                                    // centre of window g0 + l is base g0 + l + h; the seven bases start at g0 + l + h - 3
            const uint32_t first = g0 + h - 3;
            uint64_t acc = 0;                              // rolling: the low 14 bits are the current seven bases
            for (uint32_t b = 0; b < 6; ++b) acc = (acc << 2) | packed_base(ins.t.packed, (uint64_t)first + b);
            for (uint32_t l = 0; l < 32; ++l) {
                acc = (acc << 2) | packed_base(ins.t.packed, (uint64_t)first + 6 + l);
                if (sampled((uint32_t)acc & 0x3FFFu)) hits |= 1u << l;
            }
        } else if (g0 < total) {
            uint32_t sj = find_seq(ins.t.seqs, ins.t.n_seqs, g0);
            for (uint32_t l = 0; l < 32; ++l) {
                const uint32_t g = g0 + l;
                if (g >= total) break;
                while (sj + 1 < ins.t.n_seqs && ins.t.seqs[sj + 1].start <= g) ++sj;
                const SeqInfo q = ins.t.seqs[sj];
                const uint64_t fs = g - q.start;
                if (fs >= q.len || window_dots(q, fs, k) != 0) continue;
                uint32_t c = 0;
                for (uint32_t b = 0; b < 7; ++b) c = (c << 2) | packed_base(ins.t.packed, (uint64_t)g + h - 3 + b);
                if (sampled(c)) hits |= 1u << l;
            }
        }
        // the sampled windows of this thread, one at a time; the lanes of a warp go through upsert together (it votes)
#ifdef __CUDA_ARCH__
        for (;;) {
            const bool have = hits != 0;
            if (!__any_sync(0xFFFFFFFFu, have)) break;
            typename InsertBody<W>::Unit u[1];
            u[0].fwd = Key<W>(); u[0].rc = Key<W>(); u[0].h = 0; u[0].flags = 0; u[0].g = g0; u[0].valid = have;
            if (have) {
                const uint32_t l = (uint32_t)ac_ctz(hits); hits &= hits - 1; u[0].g = g0 + l;
                u[0].fwd = fetch_codes<W>(ins.t.packed, u[0].g, ins.p); u[0].rc = key_rc(u[0].fwd, ins.p);
                u[0].h = key_hash(key_select(key_is_canonical(u[0].fwd, ins.p), u[0].fwd, u[0].rc));
            }
            ins.template upsert<1>(u);
        }
#else
        for (; hits; hits &= hits - 1) {
            typename InsertBody<W>::Unit u[1];
            u[0].g = g0 + (uint32_t)ac_ctz(hits); u[0].flags = 0; u[0].valid = true;
            u[0].fwd = fetch_codes<W>(ins.t.packed, u[0].g, ins.p); u[0].rc = key_rc(u[0].fwd, ins.p);
            u[0].h = key_hash(key_select(key_is_canonical(u[0].fwd, ins.p), u[0].fwd, u[0].rc));
            ins.template upsert<1>(u);
        }
#endif
    }
};

// Extension filter.  A k-mer is an edge between two (k-1)-mer nodes: its first k-1 bases, extended on the right by its last base, and
// its last k-1 bases, extended on the left by its first.  The filter records which of a node's ten extensions (right or left, one of
// "A C G T .") some distinct k-mer makes: 3 bits per extension in ONE 64-bit word chosen by the node's hash, so that all successors of
// a k-mer (the right extensions of its last k-1 bases) are tested with one load, and all its predecessors with another.  A node is
// stored on the strand that is the smaller of M and rc M; an extension b on the right of M is the extension comp(b) on the left of
// rc M.  k - 1 is even, so M = rc M can happen: such a node holds each extension on both sides.  Keyed per node, the same k-mer enters
// from either strand.  A test that passes by chance costs a table probe; a k-mer in the table always passes.
struct ExtNode { uint64_t h; bool flip, palindrome; };
template <int W> AC_D ExtNode ext_node(const Key<W>& m, const Key<W>& m_rc) {
    const int c = key_cmp_codes(m, m_rc);
    ExtNode n; n.flip = c > 0; n.palindrome = c == 0; n.h = key_hash(key_select(n.flip, m_rc, m));
    return n;
}
AC_D uint64_t ext_word(uint64_t h, uint64_t n_words) { return ac_umul64hi(h * 0x9E3779B97F4A7C15ull, n_words); }
// extension e = 5 * side + symbol: side 0 right, 1 left; symbol 0..3 the base codes, 4 the dot
AC_D uint32_t ext_other_strand(uint32_t e) { const uint32_t s = e < 5 ? e : e - 5; return (e < 5 ? 5u : 0u) + (s == 4 ? 4u : 3u - s); }
AC_D uint64_t ext_bits(uint64_t h, uint32_t e) {
    const uint64_t x = (h ^ (e + 1) * 0xD6E8FEB86659FD93ull) * 0x9E3779B97F4A7C15ull;
    return (1ull << (x >> 58)) | (1ull << ((x >> 52) & 63)) | (1ull << ((x >> 46) & 63));
}
template <int W> AC_D void ext_add(uint64_t* filter, uint64_t n_words, const Key<W>& m, const Key<W>& m_rc, uint32_t e) {
    const ExtNode n = ext_node(m, m_rc);
    uint64_t mask = ext_bits(n.h, n.flip ? ext_other_strand(e) : e);
    if (n.palindrome) mask |= ext_bits(n.h, ext_other_strand(e));
    uint64_t* w = &filter[ext_word(n.h, n_words)];
    if ((ac_ld_volatile(w) & mask) != mask) ac_atomic_or(w, mask);
}
// The entries of the distinct k-mer `f` (rc `r`, either strand): an undotted k-mer adds both of its edges' ends; "X." and ".X" (one
// dot) add the dot as an extension of X; k-mers with more dots are never a candidate of an undotted k-mer and add nothing.
template <int W> AC_D void ext_add_kmer(uint64_t* filter, uint64_t n_words, const Key<W>& f, const Key<W>& r, const KParams& p) {
    if (f.d == 0 || f.d == -1) ext_add<W>(filter, n_words, key_prefix(f), key_suffix(r, p), f.d ? 4u : (uint32_t)f.w[W - 1] & 3u);
    if (f.d == 0 || f.d == 1) ext_add<W>(filter, n_words, key_suffix(f, p), key_prefix(r), 5u + (f.d ? 4u : key_base(f, 0, p)));
}
// Which of the symbols in `want` extend the node on `side` of the strand it was looked up on, as far as the filter can tell.
AC_D uint32_t ext_test(uint64_t word, const ExtNode& n, uint32_t side, uint32_t want) {
    uint32_t got = 0;
#pragma unroll
    for (uint32_t s = 0; s < 5; ++s) {
        const uint32_t e = 5 * side + s;
        const uint64_t m = ext_bits(n.h, n.flip ? ext_other_strand(e) : e);
        if (((want >> s) & 1u) && (word & m) == m) got |= 1u << s;
    }
    return got;
}

// Node-centric degrees (kmer_graph.rs:136-166) and the per-k-mer halves of the merge rule
// (unitig_graph.rs:192-223): outOK(K) = outdeg(K)==1 && !first(rc K); inOK(K) = indeg(K)==1 && !first(K).
template <int W> struct AdjacencyBody {
    TableView t; KParams p; bool any_dotted; const uint32_t* occupied; uint8_t* flags8;   // one thread per OCCUPIED slot (full warps)
    const uint64_t* filter; uint64_t n_fwords;
    AC_D void operator()(uint64_t x) const {
        const uint64_t i = occupied[x];
        const Slot e = t.slots[i];
        const uint32_t aux = slot_flags(e);
        const Key<W> f = window_key<W>(t, slot_gpos(e, t.gb), slot_dotted(e, t.gb), p);
        const Key<W> r = key_rc(f, p);
        const bool canon_fwd = key_is_canonical(f, p);
        const Key<W> c = key_select(canon_fwd, f, r), crc = key_select(canon_fwd, r, f);
        // the candidates still to probe, on the canonical strand: bit s = the successor that appends symbol s, bit 5 + s = the
        // predecessor that prepends it (symbols 0..3 the bases, 4 the dot; kmer_graph.rs:136-166)
        uint32_t out_c = 0, in_c = 0, cand;
        if (c.d == 0) {     // neighbours seen during the insert are known to exist; the others only where the filter has them
            const uint32_t obs_out = (aux >> AC_AUX_OBS_OUT_SHIFT) & 15u, obs_in = (aux >> AC_AUX_OBS_IN_SHIFT) & 15u;
            out_c = ac_popc(obs_out); in_c = ac_popc(obs_in);
            const uint32_t syms = any_dotted ? 31u : 15u;
            const ExtNode last = ext_node<W>(key_suffix(c, p), key_prefix(crc)), first = ext_node<W>(key_prefix(c), key_suffix(crc, p));
            const uint64_t w_last = filter[ext_word(last.h, n_fwords)], w_first = filter[ext_word(first.h, n_fwords)];
            cand = ext_test(w_last, last, 0, syms & ~obs_out) | ext_test(w_first, first, 1, syms & ~obs_in) << 5;
        } else {            // dotted k-mers (a handful per unrepaired sequence end): every candidate, probed.  p leading dots: any base
            const int32_t d = c.d;      // after it, a dot only if p = 1 ("X."), only a dot before it; trailing dots the other way round
            cand = (d > 0 ? 15u : 0u) | (d == 1 || d < 0 ? 16u : 0u) | (d < 0 ? 15u << 5 : 0u) | (d == -1 || d > 0 ? 16u << 5 : 0u);
        }
        for (; cand; cand &= cand - 1) {
            const uint32_t j = (uint32_t)ac_ctz(cand), s = j < 5 ? j : j - 5;
            Key<W> a = c;
            if (j < 5) { key_push_right(a, s & 3u, p); a.d = s == 4 ? (c.d > 0 ? -1 : c.d - 1) : (c.d > 0 ? c.d - 1 : c.d); }
            else { key_push_left(a, s & 3u, p); a.d = s == 4 ? (c.d < 0 ? 1 : c.d + 1) : (c.d < 0 ? c.d + 1 : c.d); }
            if (table_find<W>(t, a, key_rc(a, p), p) != AC_NONE32) { if (j < 5) ++out_c; else ++in_c; }
        }
        uint32_t bits = 0;
        if (out_c == 1 && !(aux & AC_AUX_FIRST_RC)) bits |= AC_FLAG8_OUT_OK;
        if (in_c == 1 && !(aux & AC_AUX_FIRST_CANON)) bits |= AC_FLAG8_IN_OK;
        flags8[i] = (uint8_t)bits;                   // bit0 outOK, bit1 inOK (canonical orientation)
    }
};
// Multi-GPU: only the k-mers of this rank's own windows need the flags (the boundary kernel reads them along the owned sequences and
// nothing else does).  The list is in coordinate order, so they are the stretch between the scanned claim counts of the words that
// hold the first and the last owned coordinate (a few foreign neighbours in those two words come along): range[w0] .. range[w1].
// A body of its own, so that the single-GPU kernel stays exactly what was measured.
template <int W> struct AdjacencyOwnBody {
    AdjacencyBody<W> all; const uint32_t* range; uint64_t w0, w1;
    AC_D void operator()(uint64_t x) const { x += range[w0]; if (x < range[w1]) all(x); }
};

// Where the unitig occurrences start: bit j of word w set <=> an occurrence starts at coordinate 32w+j, i.e. it is window 0 of a
// sequence or the edge from the previous window is not merged.  One thread per coordinate, a warp per word: the slot ids are read
// coalesced, the flag gathers of 32 windows are in flight together, the previous window's state comes from the lane below (lane 0
// fetches it), and a ballot assembles the word.
struct BoundaryBody {
    const uint64_t* packed; const SeqInfo* seqs; uint32_t n_seqs; uint32_t h; uint64_t g_begin, g_end;   // this rank's coordinates
    const uint32_t* pos_slot; const uint8_t* flags8; const uint8_t* interior;
    uint32_t* bmask; uint32_t* bcount;
    struct State { uint32_t slot; bool valid, first, in_ok, out_ok; };
    AC_D State state(uint64_t g, bool known_interior) const {
        State st; st.slot = 0; st.valid = false; st.first = false; st.in_ok = false; st.out_ok = false;
        if (!known_interior) {
            if (g < g_begin || g >= g_end) return st;
            const SeqInfo s = seqs[find_seq(seqs, n_seqs, g)];
            const uint64_t fs = g - s.start;
            if (fs >= s.len) return st;
            st.first = fs == 0;
        }
        st.valid = true;
        st.slot = pos_slot[g];
        const uint8_t fl = flags8[st.slot];
        const bool o = packed_base(packed, g + h) < 2;     // forward window is the stored orientation
        st.in_ok = o ? (fl & 2) : (fl & 1); st.out_ok = o ? (fl & 1) : (fl & 2);
        return st;
    }
    AC_D static bool starts(const State& me, const State& prev) {
        if (!me.valid) return false;
        const bool merged = !me.first && prev.out_ok && me.in_ok && me.slot != prev.slot;   // slot equality covers K'==K and K'==rc(K)
        return !merged;
    }
    AC_D void operator()(uint64_t g) const {
        const uint64_t g0 = g & ~31ull;
        const bool inside = interior[g0 >> 5] && g0 >= g_begin && g0 + 32 <= g_end;        // PackBody's flag: 32 windows of one sequence, none of them its first
#ifdef __CUDA_ARCH__
        const uint32_t lane = (uint32_t)g & 31u;
        State me, prev; prev.valid = true; prev.first = false; prev.in_ok = false;
        if (inside) {         // 32 windows of one sequence and the window before them: no sequence lookups; lane 0 fetches both windows' slots together
            const bool extra = lane == 0;
            const uint32_t slot = pos_slot[g], slot_b = extra ? pos_slot[g - 1] : 0u;
            const uint32_t fl = flags8[slot], fl_b = extra ? flags8[slot_b] : 0u;
            const bool o = packed_base(packed, g + h) < 2, o_b = extra && packed_base(packed, g - 1 + h) < 2;
            me.valid = true; me.first = false; me.slot = slot; me.in_ok = o ? (fl & 2u) : (fl & 1u); me.out_ok = o ? (fl & 1u) : (fl & 2u);
            prev.slot = __shfl_up_sync(0xFFFFFFFFu, slot, 1); prev.out_ok = __shfl_up_sync(0xFFFFFFFFu, (int)me.out_ok, 1) != 0;
            if (extra) { prev.slot = slot_b; prev.out_ok = o_b ? (fl_b & 1u) : (fl_b & 2u); }
        } else {
            me = state(g, false);
            prev.slot = __shfl_up_sync(0xFFFFFFFFu, me.slot, 1); prev.out_ok = __shfl_up_sync(0xFFFFFFFFu, (int)me.out_ok, 1) != 0;
            if (lane == 0 && me.valid && !me.first) prev = state(g - 1, false);               // the window before a word's first one (same sequence: me is not its first window)
        }
        const uint32_t word = __ballot_sync(0xFFFFFFFFu, starts(me, prev));
        if (lane == 0) { bmask[g0 >> 5] = word; bcount[g0 >> 5] = (uint32_t)__popc(word); }
#else
        if (g != g0) return;
        uint32_t word = 0;
        State prev = state(g0, inside);
        if (prev.valid && !prev.first) { const State before = state(g0 - 1, false); if (starts(prev, before)) word |= 1u; } else if (prev.valid) word |= 1u;
        for (uint32_t j = 1; j < 32; ++j) { const State me = state(g0 + j, inside); if (starts(me, prev)) word |= 1u << j; prev = me; }
        bmask[g0 >> 5] = word; bcount[g0 >> 5] = (uint32_t)__builtin_popcount(word);
#endif
    }
};

struct RunScatterBody {
    const uint32_t* bmask; const uint32_t* boff; uint64_t* run_start;
    AC_D void operator()(uint64_t i) const {
        uint32_t bits = bmask[i];
        uint32_t off = boff[i];
        while (bits) {
            const int b = ac_ctz(bits);
            run_start[off++] = i * 32 + (uint64_t)b;
            bits &= bits - 1;
        }
    }
};

// Per occurrence: its extent and the table slots of its first and last k-mer.
struct RunEndsLocalBody {
    const SeqInfo* seqs; uint32_t n_seqs; const uint64_t* run_start; uint64_t n_runs; const uint32_t* pos_slot;
    uint32_t* run_len; uint32_t* run_hs; uint32_t* run_ts;
    AC_D void operator()(uint64_t r) const {
        const uint64_t g0 = run_start[r];
        const SeqInfo s = seqs[find_seq(seqs, n_seqs, g0)];
        const uint64_t seq_last = s.start + s.len - 1;
        uint64_t g1 = seq_last;
        if (r + 1 < n_runs && run_start[r + 1] <= seq_last) g1 = run_start[r + 1] - 1;
        run_len[r] = (uint32_t)(g1 - g0 + 1); run_hs[r] = pos_slot[g0]; run_ts[r] = pos_slot[g1];
    }
};
// Multi-GPU: an occurrence in rank-independent terms (its end k-mers are named by their smallest occurrence, which is
// what every rank's table entry points at after the exchange), and back into this rank's slots.
struct RunExportBody {
    const uint64_t* run_start; const uint32_t* run_len; const uint32_t* run_hs; const uint32_t* run_ts; const Slot* slots; uint32_t gb; RunRec* out;
    AC_D void operator()(uint64_t r) const {
        RunRec x; x.start = (uint32_t)run_start[r]; x.len = run_len[r];
        x.head_rep = (uint32_t)slot_gpos(slots[run_hs[r]], gb); x.tail_rep = (uint32_t)slot_gpos(slots[run_ts[r]], gb);
        out[r] = x;
    }
};
struct RunImportBody {
    const RunRec* in; const uint32_t* pos_slot; uint64_t* run_start; uint32_t* run_len; uint32_t* run_hs; uint32_t* run_ts;
    uint32_t n_ranks; uint64_t first[AC_MAX_RANKS + 1]; const RunRec* src[AC_MAX_RANKS];     // n_ranks == 0: `in` is dense; else rank q's records [first[q], first[q+1]) start at src[q] (possibly a peer's memory)
    AC_D void operator()(uint64_t r) const {
        const RunRec* from = in + r;
        if (n_ranks) { uint32_t q = 0; while (q + 1 < n_ranks && first[q + 1] <= r) ++q; from = src[q] + (r - first[q]); }
        const RunRec x = *from;
        run_start[r] = x.start; run_len[r] = x.len; run_hs[r] = pos_slot[x.head_rep]; run_ts[r] = pos_slot[x.tail_rep];
    }
};
// The identity of an occurrence's unitig: a unitig is named by the smaller of the table slots of its two end k-mers
// (each canonical k-mer belongs to exactly one unitig); `dir` tells from which end this occurrence reads it.  The
// smallest occurrence index becomes the representative.
struct RunKeyBody {
    const uint64_t* packed; uint32_t h; const uint64_t* run_start; const uint32_t* run_hs; const uint32_t* run_ts;
    uint32_t* run_uk; uint8_t* run_dir; uint32_t* uid_rep;
    AC_D void operator()(uint64_t r) const {
        const uint32_t hs = run_hs[r], ts = run_ts[r];
        const uint32_t uk = hs < ts ? hs : ts;
        uint8_t dir;
        if (hs != ts) dir = hs < ts ? 0 : 1;
        else dir = packed_base(packed, run_start[r] + h) < 2 ? 0 : 1;     // single k-mer: orientation of the window itself
        run_uk[r] = uk; run_dir[r] = dir;
        ac_atomic_min(&uid_rep[uk], (uint32_t)r);
    }
};

struct RepFlagBody {
    const uint32_t* run_uk; const uint32_t* uid_rep; uint32_t* is_rep;
    AC_D void operator()(uint64_t r) const { is_rep[r] = uid_rep[run_uk[r]] == (uint32_t)r ? 1u : 0u; }
};

struct RunAssignBody {
    const uint64_t* run_start; const uint32_t* run_len; const uint32_t* run_uk; const uint8_t* run_dir;
    const uint32_t* uid_rep; const uint32_t* rep_idx; const uint32_t* run_hs; const uint32_t* run_ts; TableView t;
    uint32_t* run_unitig; DeviceUnitig* unitigs; uint32_t* slot_unitig;
    AC_D void operator()(uint64_t r) const {
        const uint32_t rep = uid_rep[run_uk[r]];
        const uint32_t j = rep_idx[rep];
        run_unitig[r] = (j << 1) | (run_dir[r] == run_dir[rep] ? 1u : 0u);
        if (rep == (uint32_t)r) {
            const uint32_t hs = run_hs[r], ts = run_ts[r];
            DeviceUnitig u;
            u.start = run_start[r]; u.len = run_len[r]; u.depth = table_depth(t, hs); u.flip = 0; u.min_d = 0;
            u.head_slot = hs; u.tail_slot = ts;
            for (int w = 0; w < AC_MAX_W; ++w) u.min_w[w] = 0;
            unitigs[j] = u;
            slot_unitig[hs] = j; slot_unitig[ts] = j;
        }
    }
};

// The distinct k-mers as a list of their slots: the windows that claimed a slot (InsertBody::claimed_bits), compacted.
struct ClaimedCountBody { const uint32_t* bits; uint64_t n_words; uint32_t* cnt; AC_D void operator()(uint64_t w) const { cnt[w] = w < n_words ? ac_popc(bits[w]) : 0u; } };
// With a filter, the same pass enters every distinct k-mer into the extension filter: its key is cut from the packed words at the
// claiming window (the same words for a warp's lanes) rather than from the occurrence its slot points at.
template <int W> struct ClaimedListBody {     // one thread per coordinate: slot ids read coalesced, a word's entries written side by side
    const uint32_t* bits; const uint32_t* off; const uint32_t* pos_slot; uint32_t* list;
    TableView t; KParams p; const uint8_t* interior; uint64_t* filter; uint64_t n_fwords;     // filter: null when only the list is wanted
    AC_D void operator()(uint64_t g) const {
        const uint32_t m = bits[g >> 5], b = (uint32_t)g & 31u;
        if (!((m >> b) & 1u)) return;
        list[off[g >> 5] + ac_popc(m & ((1u << b) - 1u))] = pos_slot[g];
        if (filter) {
            const Key<W> f = window_key<W>(t, g, !interior[g >> 5], p);
            ext_add_kmer<W>(filter, n_fwords, f, key_rc(f, p), p);
        }
    }
};
// Multi-GPU exchange of the deduplicated local tables ("k-mer buckets"): the occupied slots, by the list the insert kernel made.
struct ExportScatterBody {
    TableView t; const uint32_t* occupied; SlotRec* out;
    AC_D void operator()(uint64_t x) const { const uint64_t i = occupied[x]; SlotRec r; r.slot = t.slots[i]; r.count = table_depth(t, i); r.pad = 0; out[x] = r; }
};
// Folding another rank's entries into this rank's table: counts add, first/last flags OR, the entry keeps the smaller
// occurrence.  Every rank holds all packed sequences, so the k-mer behind a remote entry is read from `packed`.
template <int W> struct MergeBody {
    TableView t; KParams p; const SlotRec* in; uint32_t* pos_slot; unsigned long long* counters; uint32_t* claimed_bits;
    AC_D void operator()(uint64_t i) const {
        const SlotRec r = in[i];
        const uint64_t g = slot_gpos(r.slot, t.gb);
        const bool dotted = slot_dotted(r.slot, t.gb);
        const uint32_t flags = slot_flags(r.slot);
        const Key<W> fwd = window_key<W>(t, g, dotted, p);
        const Key<W> rc = key_rc(fwd, p);
        const uint64_t h = key_hash(key_is_canonical(fwd, p) ? fwd : rc);
        const uint32_t tag = make_tag(dotted, h, t.gb);
        const Slot mine = make_slot(g, tag, t.count_big ? 0u : r.count, flags, t.gb);
        if (!t.count_big && r.count >= t.alarm) counters[3] = 1;
        uint64_t slot = table_home(t, h);
        for (uint32_t probes = 0;; ++probes) {
            if (probes > 8192) { counters[2] = 1; return; }
            Slot e = ac_ld_cg(&t.slots[slot]);
            if (e == AC_EMPTY_SLOT) {
                e = ac_atomic_cas(&t.slots[slot], (Slot)AC_EMPTY_SLOT, mine);
                if (e == AC_EMPTY_SLOT) { if (t.count_big) ac_atomic_add(&t.count_big[slot], r.count); if (dotted) ac_atomic_add(&counters[1], 1ull); ac_atomic_or(&claimed_bits[g >> 5], 1u << (g & 31u)); break; }
            }
            if (slot_tag(e, t.gb) == tag) {
                const Key<W> rep = window_key<W>(t, slot_gpos(e, t.gb), dotted, p);
                if (key_eq(rep, fwd) || key_eq(rep, rc)) { slot_add_occurrence(t, slot, e, g, r.count, flags, true, counters); break; }
            }
            if (++slot == t.cap) slot = 0;
        }
        pos_slot[g] = (uint32_t)slot;
    }
};

struct ChunkCountBody {
    const DeviceUnitig* unitigs; uint32_t* nchunks;
    AC_D void operator()(uint64_t j) const { nchunks[j] = (unitigs[j].len + AC_MINCHUNK - 1) / AC_MINCHUNK; }
};

template <int W> struct MinPartial { Key<W> key; uint32_t from_rc; };

// Smallest k-mer (5-letter byte order) over both strands of AC_MINCHUNK consecutive windows of a unitig.
template <int W> struct ChunkMinBody {
    const uint64_t* packed; const SeqInfo* seqs; uint32_t n_seqs; KParams p;
    const DeviceUnitig* unitigs; uint32_t n_unitigs; const uint32_t* chunk_off; MinPartial<W>* partial;
    AC_D void operator()(uint64_t c) const {
        uint32_t lo = 0, hi = n_unitigs;       // largest j with chunk_off[j] <= c
        while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (chunk_off[mid] <= c) lo = mid; else hi = mid; }
        const DeviceUnitig u = unitigs[lo];
        const uint64_t first = (c - chunk_off[lo]) * AC_MINCHUNK;
        const uint64_t n = (u.len - first < AC_MINCHUNK) ? u.len - first : AC_MINCHUNK;
        uint64_t g = u.start + first;
        const SeqInfo s = seqs[find_seq(seqs, n_seqs, g)];
        uint64_t fs = g - s.start;
        Key<W> fwd, rc, best = Key<W>(); bool rolling = false, have = false; uint32_t best_rc = 0;
        for (uint64_t t = 0; t < n; ++t, ++g, ++fs) {
            const int32_t d = window_dots(s, fs, p.k);
            if (d != 0) { fwd = fetch_codes<W>(packed, g, p); fwd.d = d; rc = key_rc(fwd, p); rolling = false; }
            else if (!rolling) { fwd = fetch_codes<W>(packed, g, p); rc = key_rc(fwd, p); rolling = true; }
            else { const uint64_t code = packed_base(packed, g + p.k - 1); key_push_right(fwd, code, p); key_push_left(rc, 3 - code, p); }
            if (!have || key_less5(fwd, best)) { best = fwd; best_rc = 0; have = true; }
            if (key_less5(rc, best)) { best = rc; best_rc = 1; }
        }
        MinPartial<W> out; out.key = best; out.from_rc = best_rc;
        partial[c] = out;
    }
};

// The walk's seed is the smallest k-mer of both strands; the strand that holds it is the unitig's
// forward strand (unitig_graph.rs:179-185: seeds are visited in sorted order, forward = the seed).
template <int W> struct UnitigMinBody {
    const uint32_t* chunk_off; const MinPartial<W>* partial; DeviceUnitig* unitigs;
    AC_D void operator()(uint64_t j) const {
        const uint32_t c0 = chunk_off[j], c1 = chunk_off[j + 1];
        MinPartial<W> best = partial[c0];
        for (uint32_t c = c0 + 1; c < c1; ++c) { const MinPartial<W> q = partial[c]; if (key_less5(q.key, best.key)) best = q; }
        DeviceUnitig u = unitigs[j];
        u.flip = best.from_rc; u.min_d = best.key.d;
        for (int w = 0; w < W; ++w) u.min_w[w] = best.key.w[w];
        unitigs[j] = u;
    }
};

// unitig_graph.rs:234-287 create_links, as k-mer adjacency: the successors of a unitig strand's last k-mer
// are the first k-mers of the linked unitig strands (overlap k-1 on the untrimmed sequences).
template <int W> struct LinkBody {
    TableView t; KParams p; bool any_dotted;
    const DeviceUnitig* unitigs; const uint32_t* pos_slot; const uint32_t* slot_unitig;
    uint32_t* link_count; uint32_t* links;
    AC_D void operator()(uint64_t i) const {
        const uint32_t j = (uint32_t)(i >> 1), e = (uint32_t)(i & 1);
        const DeviceUnitig u = unitigs[j];
        Key<W> tail, tail_rc;
        if (e == 0) {
            const uint64_t g = u.start + u.len - 1;
            tail = fetch_codes<W>(t.packed, g, p);
            const SeqInfo s = t.seqs[find_seq(t.seqs, t.n_seqs, g)];
            tail.d = window_dots(s, g - s.start, p.k);
            tail_rc = key_rc(tail, p);
        } else {
            const uint64_t g = u.start;
            tail_rc = fetch_codes<W>(t.packed, g, p);
            const SeqInfo s = t.seqs[find_seq(t.seqs, t.n_seqs, g)];
            tail_rc.d = window_dots(s, g - s.start, p.k);
            tail = key_rc(tail_rc, p);
        }
        uint32_t n = 0;
        for_each_successor<W>(tail, tail_rc, any_dotted, p, [&](const Key<W>& a, const Key<W>& arc) {
            const uint32_t s2 = table_find<W>(t, a, arc, p);
            if (s2 == AC_NONE32) return;
            const uint32_t j2 = slot_unitig[s2];
            const DeviceUnitig v = unitigs[j2];
            // `a` heads unitig j2 read in its representative direction iff it is the forward k-mer of v's first window
            const bool a_canon = key_is_canonical(a, p);
            const bool head_fwd = v.head_slot == s2 && ((packed_base(t.packed, v.start + p.h) < 2) == a_canon);
            if (n < AC_MAX_LINKS) links[i * AC_MAX_LINKS + n] = (j2 << 1) | (head_fwd ? 0u : 1u);
            ++n;
        });
        link_count[i] = n;
    }
};

// ------------------------------------------------------------------------------------------------
// Seed order and the host-ready arrays
// ------------------------------------------------------------------------------------------------
// Seed order = ascending byte order of the seed k-mer text (kmer_graph.rs:168-173), i.e. key_less5 on the stored
// seed k-mers.  The seeds are minima, so their leading bits are heavily skewed and bucketing on them does not work;
// a bottom-up merge sort does: in every pass each element finds its place in the merged pair of runs with one binary
// search in the sibling run (thread per element, U <= ~10^6 keys, all of them L2 resident).
struct alignas(16) SortRec { uint64_t a, b; uint32_t c, d, id, pad; };     // what the sorts move around: a comparator's 24-byte key and the id it belongs to
struct SeedLess {
    const DeviceUnitig* unitigs; int W;
    typedef SortRec Key;      // a: first key word, b: second (0 for W = 1), c: leading dots, d: trailing dots
    AC_D Key load(uint32_t id) const {
        const DeviceUnitig& x = unitigs[id];
        Key k; k.id = id; k.pad = 0; k.a = x.min_w[0]; k.b = W > 1 ? x.min_w[1] : 0; k.c = x.min_d > 0 ? (uint32_t)x.min_d : 0u; k.d = x.min_d < 0 ? (uint32_t)-x.min_d : 0u;
        return k;
    }
    AC_D bool less_keys(const Key& x, const Key& y, uint32_t ia, uint32_t ib) const {
        if (x.c != y.c) return x.c > y.c;
        if (x.a != y.a) return x.a < y.a;
        if (x.b != y.b) return x.b < y.b;
        if (W > 2) return (*this)(ia, ib);             // the first 128 key bits tie: the full comparison
        return x.d > y.d;
    }
    AC_D bool operator()(uint32_t a, uint32_t b) const {
        const DeviceUnitig& x = unitigs[a]; const DeviceUnitig& y = unitigs[b];
        const int lx = x.min_d > 0 ? x.min_d : 0, ly = y.min_d > 0 ? y.min_d : 0;
        if (lx != ly) return lx > ly;
        for (int w = 0; w < W; ++w) if (x.min_w[w] != y.min_w[w]) return x.min_w[w] < y.min_w[w];
        const int tx = x.min_d < 0 ? -x.min_d : 0, ty = y.min_d < 0 ? -y.min_d : 0;
        return tx > ty;
    }
};
#define AC_SORT_LEAF 8
#define AC_SORT_WAYS 8          // runs merged per global pass: 2048 -> 16 Ki -> 128 Ki -> 1 Mi elements
// One merge pass over self-contained 32-byte records (the comparison key with the id inside): AC_SORT_WAYS sorted runs of `width`
// become one.  Every element finds how many elements of each sibling run go before it — for an earlier run those not above it, for a
// later run those strictly below it — with the binary searches in the siblings advanced in lockstep, so that their loads (one record per
// step and sibling, nothing to chase) are in flight together.  A pass costs about one search's latency; three passes sort a million.
template <class Less> struct MergeWaysBody {
    Less less; uint32_t n, width, steps; const SortRec* in; SortRec* out; uint32_t* idx_out;
    AC_D void operator()(uint64_t i) const {
        const SortRec me = in[i];
        const uint64_t run = i / width, group = run / AC_SORT_WAYS, group_start = group * AC_SORT_WAYS * (uint64_t)width;
        uint32_t lo[AC_SORT_WAYS], hi[AC_SORT_WAYS];
#pragma unroll
        for (int s = 0; s < AC_SORT_WAYS; ++s) {
            const uint64_t first = group_start + (uint64_t)s * width, last = first + width;
            lo[s] = (uint32_t)(first < n ? first : n); hi[s] = (uint32_t)(last < n ? last : n);
            if (group * AC_SORT_WAYS + s == run) hi[s] = lo[s];          // my own run: nothing to count
        }
        for (uint32_t step = 0; step < steps; ++step) {
#pragma unroll
            for (int s = 0; s < AC_SORT_WAYS; ++s) {
                if (lo[s] < hi[s]) {
                    const uint32_t mid = (lo[s] + hi[s]) >> 1;
                    const SortRec x = in[mid];
                    const bool earlier = group * AC_SORT_WAYS + s < run;
                    const bool before = earlier ? !less.less_keys(me, x, me.id, x.id) : less.less_keys(x, me, x.id, me.id);
                    if (before) lo[s] = mid + 1; else hi[s] = mid;
                }
            }
        }
        uint64_t pos = group_start + (i - run * width);
#pragma unroll
        for (int s = 0; s < AC_SORT_WAYS; ++s) {
            const uint64_t first = group_start + (uint64_t)s * width;
            if (group * AC_SORT_WAYS + s != run && first < n) pos += lo[s] - (uint32_t)first;
        }
        out[pos] = me; idx_out[pos] = me.id;
    }
};

// The first eleven merge levels inside one CTA: AC_SORT_TILE records are sorted in shared memory (insertion-sorted leaves of 8, then
// merge rounds with a block barrier instead of a launch between them; 4-way rounds were tried and lost, r2i).  Every `Less` used here is a strict total order (ties
// end at the index or an earlier position), so the result does not depend on how the sort is carried out.
#ifndef AC_EMULATE
#define AC_SORT_TILE 2048
#else
#define AC_SORT_TILE 16          // small tiles: the CPU suite's graphs then go through several merge passes
#endif
#ifndef AC_EMULATE
template <class Less> __global__ void __launch_bounds__(1024) ac_tile_sort_kernel(const Less less, uint32_t n, uint32_t* __restrict__ idx, SortRec* __restrict__ recs) {
    extern __shared__ __align__(16) unsigned char tile_smem[];
    SortRec* keys = reinterpret_cast<SortRec*>(tile_smem);                                           // [AC_SORT_TILE] the records, staged once
    uint16_t* buf0 = reinterpret_cast<uint16_t*>(tile_smem + AC_SORT_TILE * sizeof(SortRec));         // local ids, ping
    uint16_t* buf1 = buf0 + AC_SORT_TILE;                                                            // pong
    const uint32_t base = blockIdx.x * AC_SORT_TILE, count = n - base < AC_SORT_TILE ? n - base : AC_SORT_TILE;
    for (uint32_t i = threadIdx.x; i < count; i += blockDim.x) { SortRec r = less.load(base + i); r.id = base + i; r.pad = 0; keys[i] = r; }
    __syncthreads();
    auto before = [&](uint32_t x, uint32_t y) { return less.less_keys(keys[x], keys[y], base + x, base + y); };
    if (threadIdx.x < AC_SORT_TILE / AC_SORT_LEAF) {   // leaves: 8 consecutive ids per thread
        const uint32_t a = threadIdx.x * AC_SORT_LEAF, b = a + AC_SORT_LEAF < count ? a + AC_SORT_LEAF : count;
        uint16_t v[AC_SORT_LEAF];
        for (uint32_t x = a; x < b; ++x) {
            uint32_t y = x - a;
            while (y > 0 && before(x, v[y - 1])) { v[y] = v[y - 1]; --y; }
            v[y] = (uint16_t)x;
        }
        for (uint32_t x = a; x < b; ++x) buf0[x] = v[x - a];
    }
    __syncthreads();
    uint16_t* in = buf0; uint16_t* out = buf1;
    for (uint32_t width = AC_SORT_LEAF; width < count; width *= 2) {
        for (uint32_t i = threadIdx.x; i < count; i += blockDim.x) {
            const uint32_t me = in[i];
            const uint32_t run = i / width, pair_start = (run & ~1u) * width, run_start = run * width;
            const bool left = !(run & 1u);
            uint32_t lo, hi;
            if (left) { lo = run_start + width; hi = lo + width; } else { lo = pair_start; hi = run_start; }
            if (lo > count) lo = count;
            if (hi > count) hi = count;
            const uint32_t first = lo;
            while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; const bool bf = left ? before(in[mid], me) : !before(me, in[mid]); if (bf) lo = mid + 1; else hi = mid; }
            out[pair_start + (i - run_start) + (lo - first)] = (uint16_t)me;
        }
        __syncthreads();
        uint16_t* t = in; in = out; out = t;
    }
    for (uint32_t i = threadIdx.x; i < count; i += blockDim.x) { const SortRec r = keys[in[i]]; recs[base + i] = r; idx[base + i] = r.id; }
}
#endif
template <class Less> struct TileSortBody {   // emulation form: any correct sort of the tile
    Less less; uint32_t n; uint32_t* idx; SortRec* recs;
    AC_D void operator()(uint64_t c) const {
        const uint32_t a = (uint32_t)c * AC_SORT_TILE, b = a + AC_SORT_TILE < n ? a + AC_SORT_TILE : n;
        for (uint32_t x = a; x < b; ++x) {
            uint32_t y = x;
            while (y > a && less(x, idx[y - 1])) { idx[y] = idx[y - 1]; --y; }
            idx[y] = x;
        }
        for (uint32_t x = a; x < b; ++x) { SortRec r = less.load(idx[x]); r.id = idx[x]; r.pad = 0; recs[x] = r; }
    }
};
// Sorts the ids 0..n-1 by `less`; returns the buffer (a or b) that holds the result.  ra / rb: n records each.
template <class Less> static uint32_t* sort_indices(AcStream* stream, const Less& less, uint32_t n, uint32_t* a, uint32_t* b, SortRec* ra, SortRec* rb) {
    if (n == 0) return a;
    const uint64_t tiles = ((uint64_t)n + AC_SORT_TILE - 1) / AC_SORT_TILE;
#ifndef AC_EMULATE
    const size_t smem = AC_SORT_TILE * (sizeof(SortRec) + 2 * sizeof(uint16_t));
    // 32 warps on the SM: the searches are chains of dependent shared-memory loads.  The shared-memory opt-in is per device: cheap enough to repeat
    ac_launch_kernel("tile_sort", stream, ac_tile_sort_kernel<Less>, (unsigned)tiles, 1024, smem, less, n, a, ra);
#else
    ac_launch("tile_sort", stream, TileSortBody<Less>{less, n, a, ra}, tiles);
#endif
    for (uint64_t width = AC_SORT_TILE; width < n; width *= AC_SORT_WAYS) {
        uint32_t steps = 1; while ((1ull << steps) <= width) ++steps;          // a search over at most `width` elements ends within this many halvings
        ac_launch("merge_pass", stream, MergeWaysBody<Less>{less, n, (uint32_t)width, steps, ra, rb, b}, n);
        std::swap(a, b); std::swap(ra, rb);
    }
    return a;
}

// renumber_unitigs (unitig_graph.rs:295-315) for the graph as built: length descending, sequence ascending, depth descending,
// ties in creation (seed) order because the reference's sort is stable.  The first 8 bases ride along as a big-endian word.
struct NumberKeyBody {
    const UnitigRec* rec; const char* arena; uint64_t* prefix;
    AC_D void operator()(uint64_t s) const {
        const unsigned char* q = (const unsigned char*)(arena + rec[s].seq_off);
        const uint32_t m = rec[s].len < 8 ? rec[s].len : 8;
        uint64_t v = 0;
        for (uint32_t i = 0; i < m; ++i) v |= (uint64_t)q[i] << (56 - 8 * i);
        prefix[s] = v;
    }
};
struct InversePermBody { const uint32_t* order; uint32_t* pos; AC_D void operator()(uint64_t n) const { pos[order[n]] = (uint32_t)n; } };
struct NumberLess {
    const UnitigRec* rec; const uint32_t* depth; const char* arena; const uint64_t* prefix;
    const uint32_t* pos;     // ties keep the order the unitigs are in: creation order (null) or their place in an earlier numbering
    typedef SortRec Key;      // a: first 8 bases, b: position that settles ties, c: length, d: depth
    AC_D Key load(uint32_t id) const { Key k; k.id = id; k.pad = 0; k.a = prefix[id]; k.b = pos ? pos[id] : id; k.c = rec[id].len; k.d = depth[id]; return k; }
    AC_D bool less_keys(const Key& x, const Key& y, uint32_t ia, uint32_t ib) const {
        if (x.c != y.c) return x.c > y.c;
        if (x.a != y.a) return x.a < y.a;
        if (x.c > 8) return (*this)(ia, ib);           // equal length and first 8 bases: the rest of the sequences decides first
        if (x.d != y.d) return x.d > y.d;
        return x.b < y.b;
    }
    AC_D bool operator()(uint32_t a, uint32_t b) const {
        const uint32_t la = rec[a].len, lb = rec[b].len;
        if (la != lb) return la > lb;
        if (prefix[a] != prefix[b]) return prefix[a] < prefix[b];
        const char* x = arena + rec[a].seq_off; const char* y = arena + rec[b].seq_off;
        for (uint32_t i = 8; i < la; ++i) if (x[i] != y[i]) return (unsigned char)x[i] < (unsigned char)y[i];
        if (depth[a] != depth[b]) return depth[a] > depth[b];
        return pos ? pos[a] < pos[b] : a < b;
    }
};


// perm[s] = device unitig at seed position s.  Fills rank, the seed-ordered scalars and the arena space request.
struct SeedGatherBody {
    const uint32_t* perm; const DeviceUnitig* unitigs; uint32_t n;
    uint32_t* rank; uint32_t* len; uint32_t* depth; uint32_t* need; uint32_t* min_fpos; uint32_t* min_rpos;
    AC_D void operator()(uint64_t s) const {
        if (s == n) { need[s] = 0; return; }
        const uint32_t j = perm[s];
        const DeviceUnitig& u = unitigs[j];
        rank[j] = (uint32_t)s; len[s] = u.len; depth[s] = u.depth; need[s] = u.len + 2 * AC_SEQ_SLACK;
        min_fpos[s] = 0xFFFFFFFFu; min_rpos[s] = 0xFFFFFFFFu;
    }
};
struct SeqOffBody { const uint32_t* need_off; uint64_t* seq_off; AC_D void operator()(uint64_t s) const { seq_off[s] = (uint64_t)need_off[s] + AC_SEQ_SLACK; } };

// Trimmed forward sequence of every unitig (unitig.rs:120-133, 157-165): the centre base of each of its k-mers,
// reverse-complemented when the seed k-mer lies on the other strand of the representative occurrence.
struct EmitSeqBody {
    const uint64_t* packed; uint32_t h; const DeviceUnitig* unitigs; uint32_t n_unitigs; const uint32_t* chunk_off;
    const uint32_t* rank; const uint64_t* seq_off; char* arena;
    AC_D void operator()(uint64_t c) const {
        uint32_t lo = 0, hi = n_unitigs;
        while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (chunk_off[mid] <= c) lo = mid; else hi = mid; }
        const DeviceUnitig u = unitigs[lo];
        const uint64_t first = (c - chunk_off[lo]) * AC_MINCHUNK;
        const uint64_t n = (u.len - first < AC_MINCHUNK) ? u.len - first : AC_MINCHUNK;
        char* dst = arena + seq_off[rank[lo]];
        const uint64_t g0 = u.start + h + first;
        if (!u.flip) for (uint64_t t = 0; t < n; ++t) dst[first + t] = "ACGT"[packed_base(packed, g0 + t)];
        else for (uint64_t t = 0; t < n; ++t) dst[u.len - 1 - (first + t)] = "TGCA"[packed_base(packed, g0 + t)];
    }
};

AC_D UStrand seed_strand(uint32_t dev_strand, const uint32_t* rank, const DeviceUnitig* unitigs) {
    const uint32_t j = dev_strand >> 1;
    return (rank[j] << 1) | ((dev_strand & 1u) ^ (unitigs[j].flip & 1u));
}

struct LinkCountBody {
    const uint32_t* link_count; const uint32_t* rank; const DeviceUnitig* unitigs; uint32_t n_strands; uint32_t* cnt;
    AC_D void operator()(uint64_t i) const {
        if (i == n_strands) { cnt[i] = 0; return; }
        cnt[seed_strand((uint32_t)i, rank, unitigs)] = link_count[i];
    }
};

// forward_next / reverse_next in the push order of create_links (unitig_graph.rs:248-286), which iterates the unitigs
// in seed order: forward_next(a) = all b+ ascending then all b- ascending; reverse_next(a) = x- for x < a (pushed while
// iteration x handled x+ -> a+), then a- (self loop), then all b+ ascending, then x- for x > a.
struct LinkOrderBody {
    const uint32_t* link_count; const uint32_t* links; const uint32_t* rank; const DeviceUnitig* unitigs;
    const uint32_t* next_off; UStrand* next; uint32_t* prev_cnt; uint32_t* hairpins;     // hairpins: links that are their own mirror (a+ -> a-), for link_count (unitig_graph.rs:478-507)
    AC_D static uint64_t order_key(UStrand from, UStrand t) {
        const uint32_t a = from >> 1, b = t >> 1; const bool trev = t & 1;
        uint32_t phase;
        if (!(from & 1)) phase = trev ? 1 : 0;
        else phase = trev ? (b < a ? 0 : (b == a ? 1 : 3)) : 2;
        return ((uint64_t)phase << 32) | b;
    }
    AC_D void operator()(uint64_t i) const {
        const UStrand from = seed_strand((uint32_t)i, rank, unitigs);
        const uint32_t n = link_count[i];
        UStrand t[AC_MAX_LINKS];
        for (uint32_t x = 0; x < n && x < AC_MAX_LINKS; ++x) t[x] = seed_strand(links[i * AC_MAX_LINKS + x], rank, unitigs);
        for (uint32_t x = 1; x < n; ++x) {           // insertion sort, n <= 5
            const UStrand v = t[x]; const uint64_t kv = order_key(from, v); uint32_t y = x;
            while (y > 0 && order_key(from, t[y - 1]) > kv) { t[y] = t[y - 1]; --y; }
            t[y] = v;
        }
        UStrand* out = next + next_off[from];
        for (uint32_t x = 0; x < n; ++x) { out[x] = t[x]; ac_atomic_add(&prev_cnt[t[x]], 1u); if (t[x] == (from ^ 1u)) ac_atomic_add(hairpins, 1u); }
    }
};
struct PrevFillBody {   // (a,s) -> (b,t) puts (a,s) into prev(b,t)
    const uint32_t* next_off; const UStrand* next; const uint32_t* prev_off; uint32_t* cursor; UStrand* prev;
    AC_D void operator()(uint64_t from) const {
        for (uint32_t x = next_off[from]; x < next_off[from + 1]; ++x) { const UStrand t = next[x]; prev[prev_off[t] + ac_atomic_add(&cursor[t], 1u)] = (UStrand)from; }
    }
};
struct PrevSortBody {   // ascending, so that the result does not depend on the order the atomics landed in
    const uint32_t* prev_off; UStrand* prev;
    AC_D void operator()(uint64_t s) const {
        UStrand* p = prev + prev_off[s]; const uint32_t n = prev_off[s + 1] - prev_off[s];
        for (uint32_t x = 1; x < n; ++x) { const UStrand v = p[x]; uint32_t y = x; while (y > 0 && p[y - 1] > v) { p[y] = p[y - 1]; --y; } p[y] = v; }
    }
};

// The path of every sequence is the list of its occurrences (unitig_graph.rs:447-465 walks the same list through
// links and positions); forward_positions / reverse_positions only enter the output through their minimum.
struct PathBody {
    const SeqInfo* seqs; uint32_t n_seqs; const uint64_t* run_start; const uint32_t* run_len; const uint32_t* run_unitig;
    const uint32_t* rank; const DeviceUnitig* unitigs; UStrand* path; uint32_t* min_fpos; uint32_t* min_rpos;
    AC_D void operator()(uint64_t x) const {
        const uint32_t dev = run_unitig[x] >> 1, same = run_unitig[x] & 1;
        const uint32_t s = rank[dev];
        const bool plus = (same ^ (unitigs[dev].flip & 1u)) != 0;
        path[x] = (s << 1) | (plus ? 0u : 1u);
        const uint64_t g = run_start[x];
        const SeqInfo q = seqs[find_seq(seqs, n_seqs, g)];
        const uint32_t fs = (uint32_t)(g - q.start), mirrored = q.len - fs - run_len[x];   // kmer_graph.rs:103-108
        ac_atomic_min(&min_fpos[s], plus ? fs : mirrored);
        ac_atomic_min(&min_rpos[s], plus ? mirrored : fs);
    }
};
struct PackRecBody {   // structure-of-arrays -> the host's 32-byte records
    const uint64_t* seq_off; const uint32_t* len; const uint32_t* min_fpos; const uint32_t* min_rpos; UnitigRec* rec;
    AC_D void operator()(uint64_t s) const {
        UnitigRec r; r.seq_off = seq_off[s]; r.len = len[s]; r.min_fpos = min_fpos[s]; r.min_rpos = min_rpos[s];
        r.room_before = AC_SEQ_SLACK; r.room_after = AC_SEQ_SLACK; r.flags = 0;
        rec[s] = r;
    }
};
// ---- expand_repeats work list on the device (graph_simplification.rs:43-86, 190-280): everything below is decided by links,
// paths and fixed sets; host_graph.cpp holds the same logic for graphs that were edited on the host ----
struct FixedSeedBody {      // the ends of every sequence path are fixed (:199-208)
    const uint64_t* path_off; const UStrand* path; uint8_t* fixed_start; uint8_t* fixed_end;
    AC_D void operator()(uint64_t i) const {
        if (path_off[i + 1] == path_off[i]) return;
        const UStrand first = path[path_off[i]], last = path[path_off[i + 1] - 1];
        if (!(first & 1u)) fixed_start[first >> 1] = 1; else fixed_end[first >> 1] = 1;
        if (!(last & 1u)) fixed_end[last >> 1] = 1; else fixed_start[last >> 1] = 1;
    }
};
struct FixedSpreadBody {    // upstream of a fixed start the end is fixed, downstream of a fixed end the start is (:213-227); reads the seeds only
    const uint8_t* seed_start; const uint8_t* seed_end; const uint32_t* next_off; const UStrand* next; const uint32_t* prev_off; const UStrand* prev;
    uint8_t* fixed_start; uint8_t* fixed_end;
    AC_D void operator()(uint64_t u) const {
        const uint32_t s = (uint32_t)u << 1;
        if (seed_start[u]) for (uint32_t x = prev_off[s]; x < prev_off[s + 1]; ++x) { const UStrand up = prev[x]; if (!(up & 1u)) fixed_end[up >> 1] = 1; else fixed_start[up >> 1] = 1; }
        if (seed_end[u]) for (uint32_t x = next_off[s]; x < next_off[s + 1]; ++x) { const UStrand down = next[x]; if (!(down & 1u)) fixed_start[down >> 1] = 1; else fixed_end[down >> 1] = 1; }
    }
};
struct CandidateView {
    const uint32_t* order; const uint32_t* next_off; const UStrand* next; const uint32_t* prev_off; const UStrand* prev;
    const uint8_t* fixed_start; const uint8_t* fixed_end;
    // get_exclusive_inputs / outputs with the guards of expand_repeats (:64-84, :233-280) for the unitig at position n of the graph order
    AC_D bool eligible(uint32_t idx, uint32_t side) const {
        const UStrand self = idx << 1;
        const uint32_t* off = side == 0 ? prev_off : next_off; const UStrand* lst = side == 0 ? prev : next;
        const uint32_t* back_off = side == 0 ? next_off : prev_off; const UStrand* back = side == 0 ? next : prev;
        const uint32_t gn = off[self + 1] - off[self];
        if (gn < 2 || (side == 0 ? fixed_start[idx] : fixed_end[idx])) return false;
        for (uint32_t a = 0; a < gn; ++a) {
            const UStrand p = lst[off[self] + a];
            if (back_off[p + 1] - back_off[p] != 1 || back[back_off[p]] != self || (p >> 1) == idx) return false;
            const bool rev = p & 1u;
            if (side == 0 ? ((!rev && fixed_end[p >> 1]) || (rev && fixed_start[p >> 1])) : ((!rev && fixed_start[p >> 1]) || (rev && fixed_end[p >> 1]))) return false;
        }
        return true;
    }
};
struct CandidateFlagBody {  // one thread per (graph position, side), in the reference's iteration order: unitig by unitig, inputs side first
    CandidateView v; uint32_t n; uint32_t* flag;
    AC_D void operator()(uint64_t x) const {
        if (x == 2ull * n) { flag[x] = 0; return; }
        flag[x] = v.eligible(v.order[x >> 1], (uint32_t)(x & 1)) ? 1u : 0u;
    }
};
struct CandidateFillBody {
    CandidateView v; const uint32_t* flag_in; const uint32_t* index; ExpandCandidate* cands; int32_t* cand_at;
    AC_D void operator()(uint64_t x) const {
        const uint32_t idx = v.order[x >> 1], side = (uint32_t)(x & 1);
        const bool is_cand = index[x + 1] != index[x];
        cand_at[2 * (size_t)idx + side] = is_cand ? (int32_t)index[x] : -1;
        if (!is_cand) return;
        const UStrand self = idx << 1;
        const uint32_t* off = side == 0 ? v.prev_off : v.next_off; const UStrand* lst = side == 0 ? v.prev : v.next;
        ExpandCandidate c; c.idx = idx; c.side = (uint16_t)side; c.gn = (uint16_t)(off[self + 1] - off[self]);
        for (uint32_t a = 0; a < 6; ++a) c.src[a] = a < c.gn ? lst[off[self] + a] : 0u;
        cands[index[x]] = c;
        (void)flag_in;
    }
};
struct DependentsBody {     // host_graph.cpp compute_dependents
    const uint32_t* next_off; const UStrand* next; const uint32_t* prev_off; const UStrand* prev; const int32_t* cand_at; ExpandDeps* deps;
    AC_D void operator()(uint64_t u) const {
        ExpandDeps d;
        d.c[0] = cand_at[2 * u]; d.c[1] = cand_at[2 * u + 1];
        for (uint32_t rev = 0; rev < 2; ++rev) {
            const UStrand s = ((uint32_t)u << 1) | rev;
            const bool one_next = next_off[s + 1] - next_off[s] == 1, one_prev = prev_off[s + 1] - prev_off[s] == 1;
            d.c[2 + 2 * rev] = (one_next && !(next[next_off[s]] & 1u)) ? cand_at[2 * (size_t)(next[next_off[s]] >> 1)] : -1;
            d.c[3 + 2 * rev] = (one_prev && !(prev[prev_off[s]] & 1u)) ? cand_at[2 * (size_t)(prev[prev_off[s]] >> 1) + 1] : -1;
        }
        deps[u] = d;
    }
};
AC_D char ac_complement(char c) { return c == 'A' ? 'T' : c == 'T' ? 'A' : c == 'C' ? 'G' : c == 'G' ? 'C' : c; }
struct CommonLengthBody {   // get_common_end_seq (:298-312) for side 0, get_common_start_seq (:283-295) for side 1: length only
    const ExpandCandidate* cands; const UnitigRec* rec; const char* arena; uint32_t* spec_len;
    AC_D char at(UStrand s, uint32_t side, uint32_t i) const {
        const UnitigRec& r = rec[s >> 1]; const char* p = arena + r.seq_off;
        const bool at_back = (side == 0) != (bool)(s & 1u);
        const char b = at_back ? p[r.len - 1 - i] : p[i];
        return (s & 1u) ? ac_complement(b) : b;
    }
    AC_D void operator()(uint64_t ci) const {
        const ExpandCandidate& cd = cands[ci];
        uint32_t c = rec[cd.src[0] >> 1].len;
        for (uint32_t a = 1; a < cd.gn; ++a) {
            const uint32_t la = rec[cd.src[a] >> 1].len;
            if (la < c) c = la;
            uint32_t m = 0;
            while (m < c && at(cd.src[a], cd.side, m) == at(cd.src[0], cd.side, m)) ++m;
            c = m;
        }
        spec_len[ci] = c;
    }
};

// ---- expand_repeats on the device (fused builds; host_graph.cpp apply_candidate is the model) ----
// Two candidates conflict when they share a unitig; level = 1 + the highest level of an earlier conflicting candidate.  The earlier
// readers of a unitig are its deps entries, so the levels are the fixed point of "1 + max over predecessors" (longest path in a DAG
// whose edges point to higher indices), reached in as many relaxation rounds as there are levels.
struct LevelPredBody {
    const ExpandCandidate* cands; const ExpandDeps* deps; int32_t* pred;     // [7 * n]
    AC_D int32_t before(uint32_t u, int32_t ci) const { int32_t best = -1; for (int x = 0; x < 6; ++x) { const int32_t d = deps[u].c[x]; if (d < ci && d > best) best = d; } return best; }
    AC_D void operator()(uint64_t ci) const {
        const ExpandCandidate& cd = cands[ci];
        pred[ci * 7] = before(cd.idx, (int32_t)ci);
        for (uint32_t a = 0; a < 6; ++a) pred[ci * 7 + 1 + a] = a < cd.gn ? before(cd.src[a] >> 1, (int32_t)ci) : -1;
    }
};
struct LevelRelaxBody {
    const int32_t* pred; uint32_t* level; uint32_t* changed_and_max;       // [0] set when a level moved, [1] highest level seen
    AC_D void operator()(uint64_t ci) const {
        uint32_t lv = 0;
        for (int x = 0; x < 7; ++x) { const int32_t q = pred[ci * 7 + x]; if (q >= 0) { const uint32_t l = ac_ld_volatile(&level[q]); if (l > lv) lv = l; } }
        if (lv + 1 != level[ci]) { level[ci] = lv + 1; changed_and_max[0] = 1; }
        ac_atomic_max(&changed_and_max[1], lv + 1);
    }
};
struct RelocBoundBody {      // room the pass can ask for at most: every candidate may move its destination once, by no more than its shortest source
    const ExpandCandidate* cands; const UnitigRec* rec; const int32_t* cand_at; unsigned long long* bound;
    AC_D uint32_t shortest(const ExpandCandidate& cd) const { uint32_t m = 0xFFFFFFFFu; for (uint32_t a = 0; a < cd.gn; ++a) { const uint32_t l = rec[cd.src[a] >> 1].len; if (l < m) m = l; } return m; }
    AC_D unsigned long long bound_of(uint64_t ci) const {
        const ExpandCandidate& cd = cands[ci];
        const int32_t other = cand_at[2 * (size_t)cd.idx + (cd.side ^ 1u)];
        const unsigned long long mine = shortest(cd), partner = other >= 0 ? shortest(cands[other]) : 0;
        return (unsigned long long)rec[cd.idx].len + mine + 2 * partner + 10ull * AC_SEQ_SLACK + 64;
    }
    AC_D void operator()(uint64_t ci) const {
        ac_atomic_add(bound + (ci & (AC_BOUND_STRIPES - 1)), bound_of(ci));        // striped: one hot address would serialise in its L2 slice
    }
};
// The relaxation to its fixed point in ONE cooperative launch: a grid barrier per round instead of a launch and a host round trip.
struct LevelsCoopBody {
    const int32_t* pred; uint32_t* level; uint32_t* flags; uint64_t n;      // flags: [0..2] "a level moved" (round-robin, zeroed), [3] highest level, [4] did not settle
    template <class Sync> AC_D void operator()(uint64_t tid, uint64_t nt, Sync& sync) const {
        for (uint32_t round = 0;; ++round) {
            uint32_t* changed = flags + round % 3;
            if (tid == 0) flags[(round + 1) % 3] = 0;
            for (uint64_t ci = tid; ci < n; ci += nt) {
                uint32_t lv = 0;
                for (int x = 0; x < 7; ++x) { const int32_t q = pred[ci * 7 + x]; if (q >= 0) { const uint32_t l = ac_ld_volatile(&level[q]); if (l > lv) lv = l; } }
                if (lv + 1 != level[ci]) { level[ci] = lv + 1; *changed = 1; }
                ac_atomic_max(&flags[3], lv + 1);
            }
            sync();
            if (!ac_ld_volatile(changed)) return;
            if (round > 100000) { if (tid == 0) flags[4] = 1; return; }
        }
    }
};
// A strand of bases read without materialising it (UnitigStrand::get_seq): byte i is base[i * step], complemented when comp.
struct StrandCursor { const char* base; int32_t step; uint32_t comp; };
AC_D char cursor_at(const StrandCursor& c, uint32_t i) { const char b = c.base[(int64_t)i * c.step]; return c.comp ? ac_complement(b) : b; }
// The byte loops of a candidate, shared by the warp: the candidates of one level are scattered over the threads, so a warp seldom holds
// more than one or two active lanes — and each of those would walk hundreds of bases alone.  Every lane calls these functions (active
// or not); the lanes that own a job publish it and all 32 work through the jobs one after another.  Under emulation: plain loops.
AC_D uint32_t warp_first_mismatch(bool have, const StrandCursor& x, const StrandCursor& y, uint32_t limit) {     // owner lanes get their own result
#ifdef __CUDA_ARCH__
    uint32_t mine = limit;
    const uint32_t lane = threadIdx.x & 31u;
    for (unsigned jobs = __ballot_sync(0xFFFFFFFFu, have); jobs; jobs &= jobs - 1) {
        const int o = __ffs((int)jobs) - 1;
        StrandCursor a, b;
        a.base = (const char*)__shfl_sync(0xFFFFFFFFu, (unsigned long long)x.base, o); a.step = __shfl_sync(0xFFFFFFFFu, x.step, o); a.comp = __shfl_sync(0xFFFFFFFFu, x.comp, o);
        b.base = (const char*)__shfl_sync(0xFFFFFFFFu, (unsigned long long)y.base, o); b.step = __shfl_sync(0xFFFFFFFFu, y.step, o); b.comp = __shfl_sync(0xFFFFFFFFu, y.comp, o);
        const uint32_t n = __shfl_sync(0xFFFFFFFFu, limit, o);
        uint32_t found = n;
        for (uint32_t i0 = 0; i0 < n; i0 += 32) {
            const uint32_t i = i0 + lane;
            const bool differs = i < n && cursor_at(a, i) != cursor_at(b, i);
            const unsigned m = __ballot_sync(0xFFFFFFFFu, differs);
            if (m) { found = i0 + (uint32_t)(__ffs((int)m) - 1); break; }
        }
        if ((int)lane == o) mine = found;
    }
    return mine;
#else
    if (!have) return limit;
    uint32_t m = 0;
    while (m < limit && cursor_at(x, m) == cursor_at(y, m)) ++m;
    return m;
#endif
}
AC_D void warp_copy(bool have, char* dst, const StrandCursor& src, uint32_t n) {      // dst[i] = src[i] for i < n, for every lane that has a job
#ifdef __CUDA_ARCH__
    const uint32_t lane = threadIdx.x & 31u;
    for (unsigned jobs = __ballot_sync(0xFFFFFFFFu, have); jobs; jobs &= jobs - 1) {
        const int o = __ffs((int)jobs) - 1;
        StrandCursor a;
        a.base = (const char*)__shfl_sync(0xFFFFFFFFu, (unsigned long long)src.base, o); a.step = __shfl_sync(0xFFFFFFFFu, src.step, o); a.comp = __shfl_sync(0xFFFFFFFFu, src.comp, o);
        char* d = (char*)__shfl_sync(0xFFFFFFFFu, (unsigned long long)dst, o);
        const uint32_t m = __shfl_sync(0xFFFFFFFFu, n, o);
        for (uint32_t i = lane; i < m; i += 32) d[i] = cursor_at(a, i);
    }
    __syncwarp();
#else
    if (have) for (uint32_t i = 0; i < n; ++i) dst[i] = cursor_at(src, i);
#endif
}

struct ApplyLevelBody {      // graph_simplification.rs:64-84 for the candidates of one level; within a level no two of them share a unitig
    const ExpandCandidate* cands; const ExpandDeps* deps; const uint32_t* level; uint32_t this_level; const uint32_t* spec_len;
    UnitigRec* rec; char* arena; unsigned long long* arena_used; unsigned long long* total_shifted; uint64_t* dirty; uint8_t* exhausted;
    bool all_due;            // the first pass visits every candidate; later passes only those on the work list
    unsigned long long* total_removed;   // bases the graph lost: every source gives up the piece, the destination gains it once
    // Marks per level, so that a later pass can step over the levels nobody is due on (SimplifyCoopBody): [level] counts of the marks that
    // THIS pass will still reach (the marked candidate sits on a later level) and of those left to the next pass.  Counts only ever say
    // "somebody may be due"; the dirty bits stay the truth.
    uint32_t* due_cur = nullptr; uint32_t* due_next = nullptr;
    AC_D void count_mark(uint32_t cnd) const {
        const uint32_t lv = level[cnd];
        uint32_t* counts = !all_due && lv > this_level ? due_cur : due_next;     // chosen by value: a choice between the two addresses spills
        ac_atomic_add(counts + lv, 1u);
    }
    // strand s read from the end that candidate side `side` compares: its last bases backwards (inputs, side 0) or its first bases (outputs)
    AC_D StrandCursor cursor(UStrand s, uint32_t side) const {
        const UnitigRec& r = rec[s >> 1]; const char* p = arena + r.seq_off;
        const bool at_back = (side == 0) != (bool)(s & 1u);
        StrandCursor c; c.base = at_back ? p + r.len - 1 : p; c.step = at_back ? -1 : 1; c.comp = s & 1u;
        return c;
    }
    AC_D void mark(int32_t cnd, bool hard, int32_t below) const {
        if (cnd < 0 || cnd >= below || (!hard && exhausted[cnd])) return;
        ac_atomic_or(&dirty[(size_t)cnd >> 6], (uint64_t)1 << (cnd & 63));
        count_mark((uint32_t)cnd);
    }
    // Every lane of a warp calls this together (ci may lie beyond the list: such a lane only helps).
    AC_D void operator()(uint64_t ci, uint64_t n) const {
        bool active = ci < n && level[ci] == this_level;
        if (active && !all_due) {
            const uint64_t bit = (uint64_t)1 << (ci & 63);
            if (!(ac_ld_volatile(&dirty[ci >> 6]) & bit)) active = false;
            else ac_atomic_and(&dirty[ci >> 6], ~bit);
        }
#ifdef __CUDA_ARCH__
        if (!__any_sync(0xFFFFFFFFu, active)) return;       // nothing for this warp at this level: most warps in most levels of the later passes
#else
        if (!active) return;
#endif
        ExpandCandidate cd; cd.idx = 0; cd.side = 0; cd.gn = 0;
        if (active) cd = cands[ci];
        const uint32_t idx = cd.idx, gn = cd.gn, side = cd.side;
        bool dup = false, pristine = all_due; uint32_t min_len = 0xFFFFFFFFu;
        for (uint32_t a = 0; a < gn; ++a) {
            const uint32_t s = cd.src[a] >> 1;
            if (rec[s].len < min_len) min_len = rec[s].len;
            if (rec[s].flags) pristine = false;
            for (uint32_t b = 0; b < a; ++b) if (s == (cd.src[b] >> 1)) dup = true;
        }
        // get_common_end_seq / get_common_start_seq (:283-312) on the graph as it is now, unless the comparison made before the pass still holds
        uint32_t common_len = 0;
        const bool compare = active && !pristine;
        if (active) common_len = pristine ? spec_len[ci] : rec[cd.src[0] >> 1].len;
        const StrandCursor first = active ? cursor(cd.src[0], side) : StrandCursor{nullptr, 0, 0};
        for (uint32_t a = 1; a < 6; ++a) {                 // the warp walks the source lists in step: lane-uniform trip count
            const bool have = compare && a < gn;
            StrandCursor other = first;
            if (have) { const uint32_t la = rec[cd.src[a] >> 1].len; if (la < common_len) common_len = la; other = cursor(cd.src[a], side); }
            const uint32_t m = warp_first_mismatch(have, other, first, common_len);
            if (have) common_len = m;
        }
        uint32_t c = common_len;
        if (c > 0) { const uint32_t cap = (min_len - 1) / (dup ? 2u : 1u); if (cap < c) c = cap; }      // avoid_zero_len_unitigs (:141-158)
        const uint32_t min_pos = active ? (side == 0 ? rec[idx].min_fpos : rec[idx].min_rpos) : 0;
        if (c > 0) { if (min_pos == 0) c = 0; else if (min_pos - 1 < c) c = min_pos - 1; }               // avoid_start_of_path (:161-181)
        if (active) exhausted[ci] = c == common_len;
        const bool moving = active && c > 0;
        UnitigRec d = rec[moving ? idx : 0];
        // move the destination where there is room
        const bool relocate = moving && (side == 0 ? d.room_before < c : d.room_after < c);
        StrandCursor old_seq{arena + d.seq_off, 1, 0};
        if (relocate) {
            const uint32_t before = side == 0 ? c + 4 * AC_SEQ_SLACK : (d.room_before > AC_SEQ_SLACK ? d.room_before : AC_SEQ_SLACK);
            const uint32_t after = side == 0 ? (d.room_after > AC_SEQ_SLACK ? d.room_after : AC_SEQ_SLACK) : c + 4 * AC_SEQ_SLACK;
            const unsigned long long at_off = ac_atomic_add(arena_used, (unsigned long long)before + d.len + after);
            d.seq_off = at_off + before; d.room_before = before; d.room_after = after;
        }
        warp_copy(relocate, arena + d.seq_off, old_seq, d.len);
        // shift_sequence_1 (:89-116): the common end of the inputs becomes the start of this unitig; shift_sequence_2 (:119-138): the common
        // start of the outputs becomes its end
        StrandCursor piece = first;
        if (moving && side == 0) { piece.base = first.base + (int64_t)(c - 1) * first.step; piece.step = -first.step; }      // byte j of the piece is compared byte c-1-j
        warp_copy(moving, side == 0 ? arena + d.seq_off - c : arena + d.seq_off + d.len, piece, c);
        if (!moving) return;
        for (uint32_t a = 0; a < gn; ++a) {                // the sources lose the piece (unitig.rs:216-232)
            UnitigRec& r = rec[cd.src[a] >> 1];
            const bool rev = cd.src[a] & 1u;
            if (side == 0) { if (!rev) { r.min_rpos += c; r.len -= c; r.room_after += c; } else { r.min_fpos += c; r.len -= c; r.seq_off += c; r.room_before += c; } }
            else           { if (!rev) { r.min_fpos += c; r.len -= c; r.seq_off += c; r.room_before += c; } else { r.min_rpos += c; r.len -= c; r.room_after += c; } }
            r.flags = 1;
        }
        if (side == 0) { d.seq_off -= c; d.room_before -= c; d.len += c; d.min_fpos -= c; }            // add_seq_to_start / add_seq_to_end (unitig.rs:234-248)
        else { d.room_after -= c; d.len += c; d.min_rpos -= c; }
        d.flags = 1;
        rec[idx] = d;
        // who has to look again: in the first pass only candidates already visited (all others are still to come); later, anyone —
        // a marked candidate conflicts with this one, so it sits on another level: a later one is still reached in this pass
        const int32_t below = all_due ? (int32_t)ci : 0x7FFFFFFF;
        { const ExpandDeps& dd = deps[idx]; const bool grew_start = side == 0;
          mark(dd.c[3], grew_start, below); mark(dd.c[4], grew_start, below); mark(dd.c[2], !grew_start, below); mark(dd.c[5], !grew_start, below); }
        for (uint32_t a = 0; a < gn; ++a) {
            const ExpandDeps& ds = deps[cd.src[a] >> 1];
            const bool trimmed_end = (side == 0) != (bool)(cd.src[a] & 1u);
            if (trimmed_end) { mark(ds.c[3], false, below); mark(ds.c[4], false, below); mark(ds.c[1], false, below); }
            else { mark(ds.c[2], false, below); mark(ds.c[5], false, below); mark(ds.c[0], false, below); }
        }
        if (c != common_len) { ac_atomic_or(&dirty[(size_t)ci >> 6], (uint64_t)1 << (ci & 63)); count_mark((uint32_t)ci); }      // capped: look again next pass (its own level: counted for the next pass)
        ac_atomic_add(total_shifted, (unsigned long long)c);
        ac_atomic_add(total_removed, (unsigned long long)c * (gn - 1));
    }
};

// `while expand_repeats() > 0 {}` in ONE cooperative launch: every pass walks the levels in order with a grid barrier between them, then
// adds up the room the NEXT pass may ask for (only candidates left on the work list can act in it) and goes on while bases moved and
// the arena can take that much.  Counters (c64): [0] arena bump, [3 + 2 stripes] bases the graph lost — both running totals — and two
// sets, used by alternate passes, of { bases moved, bound stripes, candidates left }: set q lives at c64 + AC_PASS_SET(q).  A pass adds
// to its own set and, once everybody is past its first barrier (so nobody still reads the other set), thread 0 zeroes the other one for
// the pass after it: no barrier is spent on resetting counters.  res: [0] bases the last pass moved, [1] bases moved at all, [2] passes
// made by this launch, [3] the next pass's bound, [4] candidates it left, [5] the set that pass must use, [6] the arena bump.
#define AC_PASS_SET_WORDS (AC_BOUND_STRIPES + 3)
#define AC_PASS_SET(q) (1 + (q) * AC_PASS_SET_WORDS)          // [+0] bases moved, [+1 .. +stripes] bound, [+1+stripes] candidates left, [+2+stripes] arena bump once the levels are through
#define AC_PASS_REMOVED (1 + 2 * AC_PASS_SET_WORDS)
#define AC_PASS_WORDS (2 + 2 * AC_PASS_SET_WORDS)
struct SimplifyCoopBody {
    ApplyLevelBody apply; RelocBoundBody next_bound; uint64_t n; const uint32_t* n_levels;
    unsigned long long* c64; unsigned long long* res; uint64_t arena_cap; uint32_t first_set; bool first_is_pass_one;
    // Levels nobody is due on are stepped over without a barrier (later passes touch few of them: BASELINE config 2 walks 47 of its
    // 6 x 14 levels).  due: three sets of per-level mark counts (stride due_stride), used in rotation — the pass reads `cur`, marks for the
    // pass after it go to `next`, and the set the pass before read is cleared for re-use once everybody is past this pass's first barrier.
    // Every thread takes the same decision at a level: marks into cur[l] are only made while a level below l is worked on, and a barrier
    // lies between that and the first look at cur[l].  The last level is never skipped, so that every pass has a barrier.
    uint32_t* due; uint32_t due_stride, first_due;
    template <class Sync> AC_D void operator()(uint64_t tid, uint64_t nt, Sync& sync) const {
        const uint32_t levels = *n_levels;
        ApplyLevelBody a = apply;
        RelocBoundBody nb = next_bound;
        for (uint32_t pass = 0;; ++pass) {
            const uint32_t q = (first_set + pass) & 1u;
            unsigned long long* mine = c64 + AC_PASS_SET(q); unsigned long long* other = c64 + AC_PASS_SET(q ^ 1u);
            a.all_due = first_is_pass_one && pass == 0; a.total_shifted = mine;
            const uint32_t dq = (first_due + pass) % 3u;
            a.due_cur = due + (size_t)dq * due_stride; a.due_next = due + (size_t)((dq + 1u) % 3u) * due_stride;
            uint32_t* due_old = due + (size_t)((dq + 2u) % 3u) * due_stride;
            bool fenced = false;
            for (uint32_t l = 1; l <= levels; ++l) {
                if (!a.all_due && l < levels && ac_ld_volatile(&a.due_cur[l]) == 0) continue;
                a.this_level = l;
#ifdef AC_EMULATE
                if (getenv("AC_HOST_PROFILE")) {
                    uint64_t due = 0;
                    for (uint64_t ci = 0; ci < n; ++ci) if (a.level[ci] == l && (a.all_due || ((a.dirty[ci >> 6] >> (ci & 63)) & 1))) ++due;
                    fprintf(stderr, "[device] pass %u level %u: %llu due at its start\n", pass, l, (unsigned long long)due);
                }
#endif
                for (uint64_t base = 0; base < n; base += nt) a(base + tid, n);      // whole warps go in: a lane without a candidate still helps its warp
                sync();
                if (!fenced && tid == 0) {
                    for (uint32_t x = 0; x < AC_PASS_SET_WORDS; ++x) other[x] = 0;
                    for (uint32_t x = 0; x <= levels; ++x) due_old[x] = 0;
                }
                fenced = true;
                if (l == levels && tid == 0) mine[2 + AC_BOUND_STRIPES] = ac_ld_volatile(c64);       // nothing is relocated after the last level: the same value for every thread's decision below
            }
            nb.bound = mine + 1;
            for (uint64_t ci = tid; ci < n; ci += nt)
                if (ac_ld_volatile(&a.dirty[ci >> 6]) >> (ci & 63) & 1) {
                    ac_atomic_add(nb.bound + (ci & (AC_BOUND_STRIPES - 1)), nb.bound_of(ci));
                    ac_atomic_add(mine + 1 + AC_BOUND_STRIPES, 1ull);       // candidates left on the work list
                }
            sync();
            const unsigned long long moved = ac_ld_volatile(mine), used = ac_ld_volatile(mine + 2 + AC_BOUND_STRIPES);
            unsigned long long bound = 0;
            for (uint32_t x = 0; x < AC_BOUND_STRIPES; ++x) bound += ac_ld_volatile(mine + 1 + x);
            const bool go_on = moved != 0 && used + bound + 64 <= arena_cap && pass < 1000000u;
            if (tid == 0) { res[0] = moved; res[1] += moved; res[2] = pass + 1; res[3] = bound; res[4] = ac_ld_volatile(mine + 1 + AC_BOUND_STRIPES); res[5] = q ^ 1u; res[6] = used; res[7] = (dq + 1u) % 3u; }
            if (!go_on) return;
        }
    }
};

// ---- save_gfa on the device (fused builds; unitig_graph.rs:317-360, unitig.rs:167-171) ----
// S and L lines are written straight from the simplified, renumbered graph in HBM; the P lines carry host strings (file names,
// headers), so only their unitig lists are rendered here and the host wraps them.
AC_D uint32_t ac_put_dec(char* p, uint32_t v) {            // decimal text of v, returns its length
    char tmp[10]; uint32_t n = 0;
    do { tmp[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    for (uint32_t i = 0; i < n; ++i) p[i] = tmp[n - 1 - i];
    return n;
}
AC_D uint32_t ac_dec_len(uint32_t v) { uint32_t n = 1; while (v >= 10) { v /= 10; ++n; } return n; }
struct GfaView {
    const uint32_t* order; const uint32_t* number_of;     // order[n] = unitig with number n + 1; number_of[idx] = n
    const UnitigRec* rec; const char* arena; const uint32_t* depth; const uint32_t* next_off; const UStrand* next;
};
struct GfaSizeBody {
    GfaView v; uint32_t n_unitigs; uint32_t* s_size; uint32_t* l_size;
    AC_D void operator()(uint64_t n) const {
        if (n == n_unitigs) { s_size[n] = 0; l_size[n] = 0; return; }
        const uint32_t idx = v.order[n], nl = ac_dec_len((uint32_t)n + 1);
        s_size[n] = 2 + nl + 1 + v.rec[idx].len + 6 + ac_dec_len(v.depth[idx]) + 4;          // "S\t" num "\t" seq "\tDP:f:" depth ".00\n"
        uint32_t l = 0;
        for (uint32_t from = idx << 1; from <= (idx << 1 | 1u); ++from)
            for (uint32_t x = v.next_off[from]; x < v.next_off[from + 1]; ++x) l += nl + ac_dec_len(v.number_of[v.next[x] >> 1] + 1) + 11;   // "L\t" a "\t+\t" b "\t+" "\t0M\n"
        l_size[n] = l;
    }
};
struct GfaSegmentBody {
    GfaView v; const uint32_t* s_off; char* text;
    AC_D void operator()(uint64_t n) const {
        const uint32_t idx = v.order[n];
        char* p = text + s_off[n];
        *p++ = 'S'; *p++ = '\t'; p += ac_put_dec(p, (uint32_t)n + 1); *p++ = '\t';
        p += v.rec[idx].len;                                   // the bases are copied by GfaSequenceBody, 64 at a time
        *p++ = '\t'; *p++ = 'D'; *p++ = 'P'; *p++ = ':'; *p++ = 'f'; *p++ = ':'; p += ac_put_dec(p, v.depth[idx]);
        *p++ = '.'; *p++ = '0'; *p++ = '0'; *p++ = '\n';
    }
};
struct GfaChunkCountBody {    // 64-base pieces of every unitig's sequence, so that long unitigs are copied by many threads
    GfaView v; uint32_t n_unitigs; uint32_t* pieces;
    AC_D void operator()(uint64_t n) const { pieces[n] = n == n_unitigs ? 0u : (v.rec[v.order[n]].len + 63) / 64; }
};
struct GfaSequenceBody {
    GfaView v; uint32_t n_unitigs; const uint32_t* piece_off; const uint32_t* s_off; char* text;
    AC_D void operator()(uint64_t c) const {
        uint32_t lo = 0, hi = n_unitigs;                      // the unitig this piece belongs to: last n with piece_off[n] <= c
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (piece_off[mid] <= c) lo = mid; else hi = mid; }
        const uint32_t idx = v.order[lo], first = ((uint32_t)c - piece_off[lo]) * 64, len = v.rec[idx].len;
        const uint32_t m = len - first < 64 ? len - first : 64;
        const char* src = v.arena + v.rec[idx].seq_off + first;
        char* dst = text + s_off[lo] + 2 + ac_dec_len(lo + 1) + 1 + first;
        for (uint32_t i = 0; i < m; ++i) dst[i] = src[i];
    }
};
struct GfaLinkBody {          // get_links_for_gfa (:333-350): forward_next then reverse_next of every unitig, in numbering order
    GfaView v; const uint32_t* l_off; char* text;
    AC_D void operator()(uint64_t n) const {
        const uint32_t idx = v.order[n];
        char* p = text + l_off[n];
        for (uint32_t rev = 0; rev < 2; ++rev) {
            const uint32_t from = idx << 1 | rev;
            for (uint32_t x = v.next_off[from]; x < v.next_off[from + 1]; ++x) {
                const UStrand to = v.next[x];
                *p++ = 'L'; *p++ = '\t'; p += ac_put_dec(p, (uint32_t)n + 1); *p++ = '\t'; *p++ = rev ? '-' : '+'; *p++ = '\t';
                p += ac_put_dec(p, v.number_of[to >> 1] + 1); *p++ = '\t'; *p++ = (to & 1u) ? '-' : '+'; *p++ = '\t'; *p++ = '0'; *p++ = 'M'; *p++ = '\n';
            }
        }
    }
};
struct PathLastBody { const uint64_t* path_off; uint8_t* last; AC_D void operator()(uint64_t i) const { if (path_off[i + 1] > path_off[i]) last[path_off[i + 1] - 1] = 1; } };
// `path` holds seed-order unitig strands and number_of maps them to final numbers; with number_of == nullptr the entries are tokens
// already: (final number - 1) << 1 | strand (what a rank that owns the sequences, but not the graph, is sent: PathTokenBody).
AC_D uint32_t path_number(const UStrand* path, const uint32_t* number_of, uint64_t x) { return (number_of ? number_of[path[x] >> 1] : path[x] >> 1) + 1; }
struct PathSizeBody {
    const UStrand* path; const uint32_t* number_of; const uint8_t* last; uint64_t steps; uint32_t* p_size;
    AC_D void operator()(uint64_t x) const { p_size[x] = x == steps ? 0u : ac_dec_len(path_number(path, number_of, x)) + 1 + (last[x] ? 0u : 1u); }   // num sign [,]
};
struct PathTokenBody {      // every occurrence's token, laid out per owning rank: rank q's occurrences [first[q], first[q+1]) go to dst + q * stride
    const UStrand* path; const uint32_t* number_of; uint32_t* dst; uint64_t stride; uint32_t n_ranks; uint64_t first[AC_MAX_RANKS + 1];
    AC_D void operator()(uint64_t x) const {
        uint32_t q = 0; while (q + 1 < n_ranks && first[q + 1] <= x) ++q;
        dst[(uint64_t)q * stride + (x - first[q])] = (number_of[path[x] >> 1] << 1) | (path[x] & 1u);
    }
};
struct PathTextBody {
    const UStrand* path; const uint32_t* number_of; const uint8_t* last; const uint32_t* p_off; char* text;
    AC_D void operator()(uint64_t x) const {
        char* p = text + p_off[x];
        p += ac_put_dec(p, path_number(path, number_of, x)); *p++ = (path[x] & 1u) ? '-' : '+';
        if (!last[x]) *p++ = ',';
    }
};
// The P line of sequence i starts at wrap_off[i] + p_off[path_off[i]] of the P section: what the earlier sequences print around their
// lists, plus all earlier list text; its list follows the prefix, its suffix follows the list (get_gfa_path_line, unitig_graph.rs:352-360).
struct PathLineView { const uint64_t* path_off; uint32_t n_seqs; const uint32_t* p_off; const uint64_t* wrap_off; const uint32_t* pre_len; const uint32_t* suf_len; const char* blob; const uint64_t* blob_off;
                      uint64_t wrap_base; };      // wrap_off counts from the first sequence of the input; a rank that prints its own sequences only starts at wrap_base
struct PathTextFullBody {
    const UStrand* path; const uint32_t* number_of; const uint8_t* last; PathLineView v; char* text;
    AC_D void operator()(uint64_t x) const {
        uint32_t lo = 0, hi = v.n_seqs;                    // the sequence whose path holds step x
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (v.path_off[mid] <= x) lo = mid; else hi = mid; }
        char* p = text + (v.wrap_off[lo] - v.wrap_base) + v.pre_len[lo] + v.p_off[x];
        p += ac_put_dec(p, path_number(path, number_of, x)); *p++ = (path[x] & 1u) ? '-' : '+';
        if (!last[x]) *p++ = ',';
    }
};
struct PathWrapBody {       // one thread per (sequence, prefix or suffix)
    PathLineView v; char* text;
    AC_D void operator()(uint64_t t) const {
        const uint32_t i = (uint32_t)(t >> 1); const bool suffix = t & 1;
        const char* src = v.blob + v.blob_off[i] + (suffix ? v.pre_len[i] : 0u);
        char* dst = text + (v.wrap_off[i] - v.wrap_base) + (suffix ? v.pre_len[i] + v.p_off[v.path_off[i + 1]] : v.p_off[v.path_off[i]]);
        const uint32_t n = suffix ? v.suf_len[i] : v.pre_len[i];
        for (uint32_t b = 0; b < n; ++b) dst[b] = src[b];
    }
};

struct PathOffBody {
    const SeqInfo* seqs; uint32_t n_seqs; const uint64_t* run_start; uint64_t n_runs; uint64_t* path_off;
    AC_D void operator()(uint64_t i) const {
        if (i == n_seqs) { path_off[i] = n_runs; return; }
        uint64_t lo = 0, hi = n_runs;               // first run with start >= seqs[i].start
        while (lo < hi) { const uint64_t mid = (lo + hi) >> 1; if (run_start[mid] < seqs[i].start) lo = mid + 1; else hi = mid; }
        path_off[i] = lo;
    }
};

// ------------------------------------------------------------------------------------------------
// End repair (compress.rs:202-236): where do the k/2-base literals of the repair patterns occur?
// ------------------------------------------------------------------------------------------------
struct NeedleSlot { uint64_t w[2]; uint32_t id; uint32_t used; };
template <int WH> struct LiteralScanBody {
    const uint64_t* packed; const SeqInfo* seqs; uint32_t n_seqs; KParams p; uint64_t total;     // p describes an h-mer (p.k == h)
    const NeedleSlot* table; uint64_t table_mask;
    LiteralHit* hits; uint64_t hit_cap; unsigned long long* n_hits;
    AC_D void operator()(uint64_t i) const {
        uint64_t g = i * 64;
        const uint64_t g1 = (g + 64 < total) ? g + 64 : total;
        uint32_t si = find_seq(seqs, n_seqs, g);
        while (g < g1) {
            const SeqInfo s = seqs[si];
            // windows of h bases that lie entirely inside the contig: padded offsets [lead, lead + len - h]
            const uint64_t lo = s.start + s.lead, hi = s.start + s.lead + s.len - p.k;     // inclusive range of window starts
            if (g > hi || s.len < p.k) { if (si + 1 >= n_seqs) return; ++si; if (seqs[si].start > g) g = seqs[si].start; continue; }
            if (g < lo) g = lo;
            if (g >= g1) return;
            const uint64_t stop = (hi + 1 < g1) ? hi + 1 : g1;
            Key<WH> key = fetch_codes<WH>(packed, g, p);
            for (;;) {
                uint64_t slot = key_hash(key) & table_mask;
                for (;;) {
                    const NeedleSlot n = table[slot];
                    if (!n.used) break;
                    bool eq = n.w[0] == key.w[0];
                    if (WH > 1) eq = eq && n.w[1] == key.w[WH - 1];
                    if (eq) { const unsigned long long at = ac_atomic_add(n_hits, 1ull); if (at < hit_cap) { LiteralHit hh; hh.needle = n.id; hh.pad = 0; hh.gpos = g; hits[at] = hh; } break; }
                    slot = (slot + 1) & table_mask;
                }
                if (++g >= stop) break;
                key_push_right(key, packed_base(packed, g + p.k - 1), p);
            }
        }
    }
};

// ------------------------------------------------------------------------------------------------
// DeviceScan (backend.h)
// ------------------------------------------------------------------------------------------------
#ifndef AC_EMULATE
#define AC_SCAN_TILE 4096
// Tiles of 4096 values, coalesced loads, warp-shuffle block scans, in ONE launch ("chained scan with decoupled look-back"): a CTA takes
// the next tile by ticket, publishes the tile's sum, finds its exclusive prefix by looking back over the tiles before it — their sums
// until one of them has its inclusive prefix out — and scans its tile from registers (out may alias in).  A state word is [scan number:30 | status:2 | value:32], so words left by earlier
// scans never match and nothing has to be cleared between scans; tickets count up for ever (the host passes where this scan's begin).
#define AC_SCAN_STATE(epoch, status, value) (((unsigned long long)(epoch) << 34) | ((unsigned long long)(status) << 32) | (unsigned long long)(value))
__global__ void __launch_bounds__(256) ac_scan_chained_kernel(const uint32_t* in, uint64_t n, uint32_t* out, unsigned long long* state, unsigned long long epoch,
                                                               unsigned long long* ticket, unsigned long long ticket_base, uint32_t n_tiles, uint32_t* total_out) {
    __shared__ uint32_t warp_tot[8];
    __shared__ uint32_t s_tile, s_prefix;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_tile = (uint32_t)(atomicAdd(ticket, 1ull) - ticket_base);
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint64_t tile0 = (uint64_t)tile * AC_SCAN_TILE;
    uint32_t v[AC_SCAN_TILE / 1024][4], t[AC_SCAN_TILE / 1024], mine = 0;
#pragma unroll
    for (int r = 0; r < AC_SCAN_TILE / 1024; ++r) {
        const uint64_t i = tile0 + (uint64_t)r * 1024 + threadIdx.x * 4;
        if (i + 3 < n) { const uint4 q = *reinterpret_cast<const uint4*>(in + i); v[r][0] = q.x; v[r][1] = q.y; v[r][2] = q.z; v[r][3] = q.w; }
        else { for (int j = 0; j < 4; ++j) v[r][j] = (i + j < n) ? in[i + j] : 0; }
        t[r] = v[r][0] + v[r][1] + v[r][2] + v[r][3]; mine += t[r];
    }
    uint32_t sum = mine;
    for (int o = 16; o; o >>= 1) sum += __shfl_down_sync(0xFFFFFFFFu, sum, o);
    if (lane == 0) warp_tot[warp] = sum;
    __syncthreads();
    if (warp == 0) {
        uint32_t total = 0;
        for (int w2 = 0; w2 < 8; ++w2) total += warp_tot[w2];
        uint32_t prefix = 0;
        if (tile > 0) {
            if (lane == 0) *(volatile unsigned long long*)&state[tile] = AC_SCAN_STATE(epoch, 1, total);
            for (int64_t first = (int64_t)tile - 1; first >= 0; first -= 32) {      // 32 predecessors at a time, nearest first
                const int64_t j = first - lane;
                unsigned long long w = AC_SCAN_STATE(epoch, 2, 0);                  // lanes past tile 0: an inclusive prefix of nothing
                if (j >= 0) do { w = *(volatile unsigned long long*)&state[j]; } while ((w >> 34) != epoch || ((w >> 32) & 3ull) == 0);
                const unsigned closed = __ballot_sync(0xFFFFFFFFu, ((w >> 32) & 3ull) == 2);
                const int stop = closed ? __ffs((int)closed) - 1 : 31;               // the nearest tile whose inclusive prefix is out
                uint32_t part = (int)lane <= stop ? (uint32_t)w : 0u;
                for (int o = 16; o; o >>= 1) part += __shfl_down_sync(0xFFFFFFFFu, part, o);
                prefix += __shfl_sync(0xFFFFFFFFu, part, 0);
                if (closed) break;
            }
        }
        if (lane == 0) {
            *(volatile unsigned long long*)&state[tile] = AC_SCAN_STATE(epoch, 2, prefix + total);
            s_prefix = prefix;
            if (tile + 1 == n_tiles && total_out) *total_out = prefix + total;
        }
    }
    __syncthreads();
    uint32_t carry = s_prefix;
#pragma unroll
    for (int r = 0; r < AC_SCAN_TILE / 1024; ++r) {
        const uint64_t i = tile0 + (uint64_t)r * 1024 + threadIdx.x * 4;
        uint32_t inc = t[r];
        for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, inc, o); if (lane >= (uint32_t)o) inc += u; }
        __syncthreads();                  // warp_tot is reused every round
        if (lane == 31) warp_tot[warp] = inc;
        __syncthreads();
        uint32_t wbase = 0, total = 0;
        for (uint32_t w2 = 0; w2 < 8; ++w2) { const uint32_t x = warp_tot[w2]; if (w2 < warp) wbase += x; total += x; }
        uint32_t e = carry + wbase + inc - t[r];
        if (i + 3 < n) { uint4 q; q.x = e; q.y = e + v[r][0]; q.z = q.y + v[r][1]; q.w = q.z + v[r][2]; *reinterpret_cast<uint4*>(out + i) = q; }
        else { for (int j = 0; j < 4; ++j) { if (i + j < n) out[i + j] = e; e += v[r][j]; } }
        carry += total;
    }
}
uint32_t DeviceScan::operator()(AcStream* st, const uint32_t* in, uint32_t* out, uint64_t n, bool want_total) {
    if (n == 0) return 0;
    const uint64_t nb = (n + AC_SCAN_TILE - 1) / AC_SCAN_TILE;
    if (nb > 0x7FFFFFFFull) throw std::runtime_error("scan too large");
    if ((nb + 4) * 8 > state.cap) {      // [0] ticket counter, [1] the total, [2..] one state word per tile; zeroed once: scan numbers start at 1
        state.ensure((nb + 4) * 8 * 2);
        ac_memset(state.p, 0, state.cap, st);
        tickets = 0;
    }
    unsigned long long* s = state.as<unsigned long long>();
    epoch = (epoch + 1) & 0x3FFFFFFFull; if (epoch == 0) epoch = 1;
    ac_launch_kernel("scan", st, ac_scan_chained_kernel, (unsigned)nb, 256, 0, in, n, out, s + 2, epoch, s, tickets, (uint32_t)nb, (uint32_t*)(s + 1));
    tickets += nb;
    uint32_t total_sum = 0;
    if (want_total) { ac_d2h(&total_sum, s + 1, sizeof(uint32_t), st); ac_sync(st); }
    return total_sum;
}
#else
uint32_t DeviceScan::operator()(AcStream* st, const uint32_t* in, uint32_t* out, uint64_t n, bool want_total) { return serial.run(st, in, out, n, want_total); }
#endif

// ------------------------------------------------------------------------------------------------
// host orchestration
// ------------------------------------------------------------------------------------------------
// Under emulation a buffer kernels write joins its owner's set when it is constructed, so poisoning reaches each one; the product keeps nothing.
#ifdef AC_EMULATE
struct ScratchSet { std::vector<DevBuf*> bufs; };
struct ScratchBuf : DevBuf { explicit ScratchBuf(ScratchSet& set) { set.bufs.push_back(this); } };
#else
struct ScratchSet {};
struct ScratchBuf : DevBuf { explicit ScratchBuf(ScratchSet&) {} };
#endif

// The stage boundaries a build records on the pipeline's stream, in that order; complete() turns pairs of them into PipelineTimings.
enum Mark {
    UPLOAD_BEGIN, UPLOAD_END,                                                          // upload()
    PACK_BEGIN, PACK_END, SAMPLE_END, INSERT_BEGIN, INSERT_END, TABLE_END,             // build_local(); INSERT_* around the last attempt's insert kernel
    RUNS_BEGIN, ADJACENCY_END, BOUNDARIES_END,                                         // runs_local()
    FINISH_BEGIN, UNITIGS_END, SEEDS_END, LINKS_END, SEED_SORT_END, WORK_LIST_END, SIMPLIFY_END, GFA_END,   // finish()
    ALL_BUT_ARENA, RESULTS_END, N_MARKS                                                // the copies to the host: all but the arena, then the arena
};
// The last stage a call completed: upload() or find_literals(), build_local(), runs_local()
enum class Stage { UPLOADED, TABLE, RUNS };

struct DevicePipeline::Impl : DeviceContext {
    uint64_t total = 0; uint32_t n_seqs = 0, k = 0, U = 0, n_chunks = 0; int W = 0;      // U, n_chunks: unitigs and their 64-base chunks (finish)
    // inputs: what upload(), set_path_line_texts() and find_literals() copy from the host
    DevBuf ascii, seqs, d_wrap_off, d_pre_len, d_suf_len, d_blob, d_blob_off, needles;
    // scratch: everything the kernels write, by the stage that sizes it
    ScratchSet scratch;
    ScratchBuf packed{scratch}, interior8{scratch}, slots{scratch}, pos_slot{scratch}, counters{scratch}, count_big{scratch}, claimed{scratch}, claimed_cnt{scratch}, occ_list{scratch},   // table
        ext_filter{scratch}, hits{scratch};
    ScratchBuf flags8{scratch}, bmask{scratch}, bcount{scratch}, boff{scratch}, run_start{scratch}, run_len{scratch}, run_hs{scratch}, run_ts{scratch};   // runs
    ScratchBuf run_uk{scratch}, run_dir{scratch}, is_rep{scratch}, rep_idx{scratch}, run_unitig{scratch}, uid_rep{scratch}, slot_unitig{scratch}, unitigs{scratch}, nchunks{scratch},   // graph
        chunk_off{scratch}, partial{scratch}, link_count{scratch}, links{scratch}, sort_a{scratch}, sort_b{scratch}, sort_ra{scratch}, sort_rb{scratch}, rank{scratch}, d_len{scratch},
        d_depth{scratch}, need{scratch}, d_seq_off{scratch}, d_min_fpos{scratch}, d_min_rpos{scratch}, d_arena{scratch}, strand_cnt{scratch}, d_next_off{scratch}, d_next{scratch},
        prev_cnt{scratch}, d_prev_off{scratch}, d_prev{scratch}, d_small{scratch}, d_path{scratch}, d_path_off{scratch}, d_rec{scratch}, num_prefix{scratch}, d_fixed{scratch}, cand_flag{scratch},
        cand_index{scratch}, d_cands{scratch}, d_cand_at{scratch}, d_deps{scratch}, d_spec{scratch};
    ScratchBuf d_pred{scratch}, d_level{scratch}, d_flagmax{scratch}, d_counters64{scratch}, d_dirty{scratch}, d_exhausted{scratch}, d_due{scratch}, d_arena2{scratch}, d_arena3{scratch},   // simplify
        d_pos{scratch}, sort_c{scratch}, sort_d{scratch};
    ScratchBuf d_pos2{scratch}, gfa_s_size{scratch}, gfa_l_size{scratch}, gfa_p_size{scratch}, gfa_pieces{scratch}, d_last{scratch}, d_totals{scratch}, d_text{scratch}, d_own_off{scratch},   // GFA, path lines
        d_own_last{scratch}, d_own_size{scratch}, d_ptext{scratch};
    ScratchBuf own_entries{scratch}, own_runs{scratch};   // exchange
    DeviceScan scan;
    PinBuf h_rec, h_depth, h_order, h_order2, h_arena, h_next_off, h_next, h_prev_off, h_prev, h_path, h_path_off, h_run_start, h_run_len;
    PinBuf h_cands, h_deps, h_spec, h_fixed, h_text, h_ptext;
#ifndef AC_EMULATE
    cudaEvent_t ev[N_MARKS];
    Impl(int device, void* stream) : DeviceContext(device, stream) { for (auto& e : ev) AC_CUDA_CHECK(cudaEventCreate(&e)); }
    ~Impl() { cudaSetDevice(device); for (auto& e : ev) cudaEventDestroy(e); }      // the buffers go first (on this device), the stream last (DeviceContext)
    void mark(Mark m) { AC_CUDA_CHECK(cudaEventRecord(ev[m], stream.s)); }
    void wait_mark(Mark m) { AC_CUDA_CHECK(cudaEventSynchronize(ev[m])); }
    float between(Mark a, Mark b) { float ms = 0; AC_CUDA_CHECK(cudaEventElapsedTime(&ms, ev[a], ev[b])); return ms; }
#else
    Impl(int device, void* stream) : DeviceContext(device, stream) {}
    void mark(Mark) {}
    void wait_mark(Mark) {}
    float between(Mark, Mark) { return 0.f; }
#endif
    bool arena_pending = false;
    const std::function<void()>* before_results = nullptr;   // -> DevicePipeline::before_results

    // pipeline state shared by the stages
    std::vector<SeqInfo> host_seqs;
    uint64_t cap = 0, n_windows = 0, n_runs = 0, g_begin = 0, g_end = 0, n_slots_used = 0, n_dotted = 0, n_fwords = 0;
    bool any_dotted = false, is_multi = false, big_counts = false;      // big_counts: depths live in count_big (a 20-bit slot count neared its end)
    Stage stage = Stage::UPLOADED;
    void require(Stage s, const char* message) const { if (stage < s) throw std::runtime_error(message); }
    TableView table_view() { return TableView{slots.as<Slot>(), cap, packed.as<uint64_t>(), seqs.as<SeqInfo>(), n_seqs, big_counts ? count_big.as<uint32_t>() : nullptr, slot_gpos_bits(total), count_alarm()}; }
    static uint32_t count_alarm() { static const uint32_t a = getenv("AC_COUNT_ALARM") ? (uint32_t)atoi(getenv("AC_COUNT_ALARM")) : AC_SLOT_COUNT_ALARM; return a; }      // test hook: a lower threshold
    template <int W> void local_w(uint32_t seq_lo, uint32_t seq_hi, bool multi);
    template <int W> void insert_w();
    uint64_t safe_cap = 0;          // 1.5 slots per window of every sequence (all ranks'): holds any input, the union of the ranks' k-mers included
    int table_attempt = 0;          // of the current build: the initial size, the safe size, the side counts (AC_HOST_PROFILE prints each)
    std::vector<std::pair<const void*, uint64_t>> merged;      // the (records, count) of every merge_entries since build_local
    template <int W> void merge_w(const void* dev_ptr, uint64_t n);
    template <int W> void runs_local_w();
    // the stages of finish(), in their order; R carries what each leaves to the next
    template <int W> void unitigs_w(PipelineResult& out);
    void host_arrays(), paths(), work_list(), simplify(), renumber(), gfa(bool split_paths);
    void results(PipelineResult& out, bool keep_positions, bool fused);
    // what a finished build leaves in HBM for pull_graph() (at once in a plain build, on request after a fused one)
    struct Pending {
        uint64_t n_links = 0, n_cands = 0;
        uint32_t* order_built = nullptr; uint32_t* final_order = nullptr; uint8_t* fix_start = nullptr;
        DevBuf* arena_src = nullptr; uint64_t arena_final = 0;
        bool any_moved = false, gfa_on_device = false, paths_split = false;
        uint64_t bases_removed = 0, gfa_bytes = 0;
    } R;
    void pull_graph(PipelineResult& out, bool keep_positions);
    std::vector<char> path_blob; std::vector<uint32_t> path_pre, path_suf; uint64_t path_wrap_total = 0;
    uint64_t uploaded_bytes = 0;
    uint64_t exp_n = 0, n_own_runs = 0; uint32_t own_seq_lo = 0, own_seq_hi = 0; bool exp_valid = false;      // exp_n: this rank's own distinct k-mers, counted before the merge
    template <int W> uint64_t list_claimed(bool with_filter);
    template <int W> uint64_t count_entries_w();
#ifdef AC_EMULATE
    // AC_EMU_POISON=1 (CPU suite): before every table build, every scratch buffer is filled with a pattern, so a kernel that reads what
    // THIS build has not written (on the GPU: leftovers of the previous build, whose slot numbers differ from run to run, while the
    // emulation reproduces them exactly) shows up on the CPU as well.
    static void fill(DevBuf* b) { static const bool on = getenv("AC_EMU_POISON") != nullptr; if (on && b->p) memset(b->p, 0xA5, b->cap); }
    void poison() { for (DevBuf* b : scratch.bufs) fill(b); for (DevBuf& b : scan.serial.level) fill(&b); }
    // and before every attempt at the table: a retry must not read what the failed attempt left
    void poison_table() { for (DevBuf* b : {&slots, &pos_slot, &claimed, &claimed_cnt, &occ_list, &count_big, &counters}) fill(b); }
#else
    void poison() {}
    void poison_table() {}
#endif
};

DevicePipeline::DevicePipeline(int device, void* stream) : impl(new Impl(device, stream)) { impl->before_results = &before_results; }
DevicePipeline::~DevicePipeline() { delete impl; }

unsigned long long DevicePipeline::kernel_launches() const { return g_ac_kernel_launches; }
DeviceContext& DevicePipeline::context() { return *impl; }

void DevicePipeline::upload(const uint8_t* ascii, uint64_t total, const SeqInfo* seqs, uint32_t n_seqs, uint32_t k, uint32_t seq_lo, uint32_t seq_hi) {
    Impl& m = *impl; m.make_current();
    if (k < 3 || (k & 1) == 0) throw std::runtime_error("k must be odd and >= 3");
    const int W = (int)((2 * k + 63) / 64);
    if (W > AC_MAX_W) throw std::runtime_error("k-mer sizes above " + std::to_string(AC_MAX_K) + " are not supported by the GPU path (no CPU fallback exists)");
    if (total >= 0xFFFFFFF0ull) throw std::runtime_error("more than 2^32 padded input bytes are not supported");
    if (n_seqs == 0 || total == 0) throw std::runtime_error("no sequences");
    m.total = total; m.n_seqs = n_seqs; m.k = k; m.W = W; m.stage = Stage::UPLOADED;
    m.host_seqs.assign(seqs, seqs + n_seqs);
    m.mark(UPLOAD_BEGIN);
    m.ascii.ensure(total);
    if (seq_lo == 0 && seq_hi >= n_seqs) { ac_h2d(m.ascii.p, ascii, total, &m.stream); m.uploaded_bytes = total; }
    else {              // a shard: only the strands of sequences [seq_lo, seq_hi); the caller's collective brings the other ranks' blocks (strand_block)
        if (seq_lo > seq_hi || seq_hi > n_seqs) throw std::runtime_error("bad sequence shard");
        const uint64_t b0 = seq_lo < n_seqs ? seqs[seq_lo].start : total, b1 = seq_hi < n_seqs ? seqs[seq_hi].start : total;
        if (b1 > b0) ac_h2d(m.ascii.as<uint8_t>() + b0, ascii + b0, b1 - b0, &m.stream);
        m.uploaded_bytes = b1 - b0;
    }
    m.seqs.ensure(n_seqs * sizeof(SeqInfo));
    ac_h2d(m.seqs.p, seqs, n_seqs * sizeof(SeqInfo), &m.stream);
    if (m.path_pre.size() == n_seqs) {       // the P-line texts (set_path_line_texts): prefix and suffix of every sequence, and where each line's share starts
        std::vector<uint64_t> wrap((size_t)n_seqs + 1, 0), boff((size_t)n_seqs + 1, 0);
        for (uint32_t i = 0; i < n_seqs; ++i) { wrap[i + 1] = wrap[i] + m.path_pre[i] + m.path_suf[i]; boff[i + 1] = wrap[i + 1]; }
        m.path_wrap_total = wrap[n_seqs];
        m.d_wrap_off.ensure(wrap.size() * 8); m.d_blob_off.ensure(boff.size() * 8); m.d_pre_len.ensure((size_t)n_seqs * 4); m.d_suf_len.ensure((size_t)n_seqs * 4); m.d_blob.ensure(m.path_blob.size() + 8);
        ac_h2d(m.d_wrap_off.p, wrap.data(), wrap.size() * 8, &m.stream); ac_h2d(m.d_blob_off.p, boff.data(), boff.size() * 8, &m.stream);
        ac_h2d(m.d_pre_len.p, m.path_pre.data(), (size_t)n_seqs * 4, &m.stream); ac_h2d(m.d_suf_len.p, m.path_suf.data(), (size_t)n_seqs * 4, &m.stream);
        if (!m.path_blob.empty()) ac_h2d(m.d_blob.p, m.path_blob.data(), m.path_blob.size(), &m.stream);
        ac_sync(&m.stream);                  // the staging vectors above are locals
    } else m.path_wrap_total = 0;
    m.mark(UPLOAD_END);
}

void DevicePipeline::set_path_line_texts(const char* blob, const uint32_t* prefix_len, const uint32_t* suffix_len, uint32_t n) {
    Impl& m = *impl;
    m.path_pre.assign(prefix_len, prefix_len + n); m.path_suf.assign(suffix_len, suffix_len + n);
    uint64_t bytes = 0; for (uint32_t i = 0; i < n; ++i) bytes += (uint64_t)prefix_len[i] + suffix_len[i];
    m.path_blob.assign(blob, blob + bytes);
}

void DevicePipeline::find_literals(const uint8_t* ascii_host, uint64_t total_bytes, const SeqInfo* host_seq, uint32_t n, uint32_t h,
                                   const uint64_t* needle_words, uint32_t n_needles, std::vector<LiteralHit>& out) {
    Impl& m = *impl; m.make_current();
    const int WH = (int)((2 * h + 63) / 64);
    if (WH > 2) throw std::runtime_error("end repair literals longer than 64 bases are not supported by the GPU path");
    const KParams p = make_kparams(h, WH);
    m.ascii.ensure(total_bytes); ac_h2d(m.ascii.p, ascii_host, total_bytes, &m.stream);
    m.seqs.ensure(n * sizeof(SeqInfo)); ac_h2d(m.seqs.p, host_seq, n * sizeof(SeqInfo), &m.stream);
    const uint64_t n_words = (total_bytes + 31) / 32;
    m.packed.ensure((n_words + 6) * sizeof(uint64_t));
    ac_memset(m.packed.as<uint64_t>() + n_words, 0, 6 * sizeof(uint64_t), &m.stream);
    ac_launch("pack", &m.stream, PackBody{m.ascii.as<uint8_t>(), total_bytes, m.packed.as<uint64_t>(), nullptr, 0, nullptr}, n_words);
    // needle table (host-built, tiny)
    uint64_t cap = 64; while (cap < 4ull * n_needles) cap <<= 1;
    std::vector<NeedleSlot> table(cap);          // all zero: no slot used
    for (uint32_t i = 0; i < n_needles; ++i) {
        Key<2> k2; k2.w[0] = needle_words[2 * i]; k2.w[1] = needle_words[2 * i + 1]; k2.d = 0;
        uint64_t hsh;
        if (WH == 1) { Key<1> k1; k1.w[0] = k2.w[1]; k1.d = 0; hsh = key_hash(k1); } else hsh = key_hash(k2);
        uint64_t slot = hsh & (cap - 1);
        while (table[slot].used) slot = (slot + 1) & (cap - 1);
        // stored the way the scan compares: w[0] = most significant word of the WH-word key, w[1] = its last word
        table[slot].w[0] = WH == 1 ? k2.w[1] : k2.w[0]; table[slot].w[1] = k2.w[1]; table[slot].id = i; table[slot].used = 1;
    }
    m.needles.ensure(cap * sizeof(NeedleSlot)); ac_h2d(m.needles.p, table.data(), cap * sizeof(NeedleSlot), &m.stream);
    m.counters.ensure(8 * sizeof(unsigned long long));
    uint64_t hit_cap = 1u << 20;
    for (;;) {
        m.hits.ensure(hit_cap * sizeof(LiteralHit));
        ac_memset(m.counters.p, 0, sizeof(unsigned long long), &m.stream);
        if (WH == 1) ac_launch("literal_scan", &m.stream, LiteralScanBody<1>{m.packed.as<uint64_t>(), m.seqs.as<SeqInfo>(), n, p, total_bytes, m.needles.as<NeedleSlot>(), cap - 1,
                                                                           m.hits.as<LiteralHit>(), hit_cap, m.counters.as<unsigned long long>()}, (total_bytes + 63) / 64);
        else ac_launch("literal_scan", &m.stream, LiteralScanBody<2>{m.packed.as<uint64_t>(), m.seqs.as<SeqInfo>(), n, p, total_bytes, m.needles.as<NeedleSlot>(), cap - 1,
                                                                     m.hits.as<LiteralHit>(), hit_cap, m.counters.as<unsigned long long>()}, (total_bytes + 63) / 64);
        unsigned long long found = 0;
        ac_d2h(&found, m.counters.p, sizeof found, &m.stream); ac_sync(&m.stream);
        if (found <= hit_cap) { out.resize(found); if (found) { ac_d2h(out.data(), m.hits.p, found * sizeof(LiteralHit), &m.stream); ac_sync(&m.stream); } break; }
        hit_cap = found + 1024;        // short literals match often: run again with room for all of them
    }
    m.stage = Stage::UPLOADED;
}

// One instantiation of every k-mer kernel per key width: W = ceil(2k / 64) words, k up to 511.
#define AC_W_CASE(fn, n, ...) case n: fn<n>(__VA_ARGS__); break;
#define AC_DISPATCH_W(fn, ...) switch (W) { AC_W_CASE(fn, 1, __VA_ARGS__) AC_W_CASE(fn, 2, __VA_ARGS__) AC_W_CASE(fn, 3, __VA_ARGS__) AC_W_CASE(fn, 4, __VA_ARGS__) \
    AC_W_CASE(fn, 5, __VA_ARGS__) AC_W_CASE(fn, 6, __VA_ARGS__) AC_W_CASE(fn, 7, __VA_ARGS__) AC_W_CASE(fn, 8, __VA_ARGS__) AC_W_CASE(fn, 9, __VA_ARGS__) AC_W_CASE(fn, 10, __VA_ARGS__) \
    AC_W_CASE(fn, 11, __VA_ARGS__) AC_W_CASE(fn, 12, __VA_ARGS__) AC_W_CASE(fn, 13, __VA_ARGS__) AC_W_CASE(fn, 14, __VA_ARGS__) AC_W_CASE(fn, 15, __VA_ARGS__) AC_W_CASE(fn, 16, __VA_ARGS__) \
    default: throw std::runtime_error("upload() must precede build()"); }

// ---- stage 1: pack + k-mer table over this rank's sequences ----
#define AC_N_COUNTERS 4          // InsertBody::counters
template <int W> void DevicePipeline::Impl::local_w(uint32_t seq_lo, uint32_t seq_hi, bool multi) {
    const KParams p = make_kparams(k, W);
    if (seq_lo > seq_hi || seq_hi > n_seqs) throw std::runtime_error("bad sequence shard");
    const SeqInfo* hs = host_seqs.data();
    if (seq_lo == seq_hi) { g_begin = g_end = 0; }       // a rank without sequences still merges, and computes the replicated stages
    else { g_begin = hs[seq_lo].start; g_end = hs[seq_hi - 1].start + hs[seq_hi - 1].len; }
    is_multi = multi; own_seq_lo = seq_lo; own_seq_hi = seq_hi; exp_valid = false;
    poison();
    // windows = total - n_seqs*(k-1); a canonical table can hold at most that many entries (all ranks' windows: after
    // the exchange every rank's table holds the k-mers of every sequence)
    n_windows = total - (uint64_t)n_seqs * (k - 1);
    cap = (n_windows + n_windows / 2 + 64 + 3) & ~3ull;      // a multiple of 4: the table is probed in groups of four slots
    if (cap >= 0xFFFFFFF0ull) throw std::runtime_error("input too large for 32-bit slot indices");

    mark(PACK_BEGIN);
    const uint64_t n_words = (total + 31) / 32;
    packed.ensure((n_words + W + 2) * sizeof(uint64_t));
    ac_memset(packed.as<uint64_t>() + n_words, 0, (W + 2) * sizeof(uint64_t), &stream);
    interior8.ensure(n_words + 8);
    ac_launch("pack", &stream, PackBody{ascii.as<uint8_t>(), total, packed.as<uint64_t>(), seqs.as<SeqInfo>(), n_seqs, interior8.as<uint8_t>()}, n_words);
    mark(PACK_END);

    // ---- size the table: distinct canonical k-mers estimated from the 1/64 of them whose hash ends in six zero bits ----
    // (sampling by hash value keeps or drops a k-mer with ALL its occurrences, so 64 x the sample's distinct count is an
    // unbiased estimate; every rank samples every sequence because after the exchange its table holds all of them.)
    const uint64_t safe_cap = cap;
    counters.ensure(AC_N_COUNTERS * sizeof(unsigned long long));
    unsigned long long hc[AC_N_COUNTERS] = {0, 0, 0, 0};
    big_counts = getenv("AC_BIG_COUNTS") != nullptr;      // test hook: take the 32-bit side array from the start
    const double load = getenv("AC_TABLE_LOAD") ? atof(getenv("AC_TABLE_LOAD")) : 0.5;
    if (load > 0 && n_windows > (1u << 16) && k >= 7) {
        const uint64_t sample_cap = (n_windows / 64 * 4 + 4096) & ~3ull;
        slots.ensure(sample_cap * sizeof(Slot));
        ac_memset(slots.p, 0xFF, sample_cap * sizeof(Slot), &stream);
        ac_memset(counters.p, 0, sizeof hc, &stream);
        const TableView sv{slots.as<Slot>(), sample_cap, packed.as<uint64_t>(), seqs.as<SeqInfo>(), n_seqs, nullptr, slot_gpos_bits(total), AC_SLOT_COUNT_ALARM};
        const InsertBody<W> sample_ins{sv, p, interior8.as<uint8_t>(), 0, 0, (uint32_t)total, false, nullptr, counters.as<unsigned long long>(), true, nullptr};
        ac_launch("sample", &stream, SampleBody<W>{sample_ins, (uint32_t)total}, ((total + 31) / 32 + 31) / 32 * 32);
        ac_d2h(hc, counters.p, sizeof hc, &stream); ac_sync(&stream);
        if (!hc[2]) {      // every rank samples every sequence, so all of them arrive at the same size
            const uint64_t est = (hc[0] + 3 * (uint64_t)std::sqrt((double)hc[0]) + 16) * 64 + (uint64_t)n_seqs * 2 * k;      // + 3 sigma, + the windows with dots it left out
            cap = std::min<uint64_t>(safe_cap, ((uint64_t)((double)est / load) + 4096 + 3) & ~3ull);
        }
    }
    mark(SAMPLE_END);
    this->safe_cap = safe_cap;
    table_attempt = 0;
    merged.clear();
    insert_w<W>();
    mark(TABLE_END);
    stage = Stage::TABLE;
}

// The table over this rank's windows at `cap`, started again at the safe size if the probe limit trips and with the counts in the side
// array if the count alarm rises.  Every attempt starts from an empty table, so nothing of a failed one is read.
template <int W> void DevicePipeline::Impl::insert_w() {
    const KParams p = make_kparams(k, W);
    const uint64_t n_words = (total + 31) / 32;
    unsigned long long hc[AC_N_COUNTERS] = {0, 0, 0, 0};
    pos_slot.ensure(total * sizeof(uint32_t));
    for (;; ++table_attempt) {
        if (table_attempt > 3) throw std::runtime_error("k-mer table build did not settle");
        if (getenv("AC_HOST_PROFILE")) fprintf(stderr, "[device] k-mer table attempt %d: capacity %llu, side counts %d\n", table_attempt, (unsigned long long)cap, (int)big_counts);
        poison_table();
        slots.ensure(cap * sizeof(Slot));
        ac_memset(slots.p, 0xFF, cap * sizeof(Slot), &stream);               // AC_EMPTY_SLOT
        if (big_counts) { count_big.ensure(cap * 4); ac_memset(count_big.p, 0, cap * 4, &stream); }
        ac_memset(counters.p, 0, sizeof hc, &stream);
        const TableView tv = table_view();
        const uint64_t g_first = g_begin & ~63ull;     // the first unit may start up to 63 coordinates before the shard: edge_unit rejects those windows
        claimed.ensure((n_words + 8) * 4); ac_memset(claimed.p, 0, (n_words + 8) * 4, &stream);
        const InsertBody<W> ins{tv, p, interior8.as<uint8_t>(), (uint32_t)g_first, (uint32_t)g_begin, (uint32_t)g_end, is_multi, pos_slot.as<uint32_t>(), counters.as<unsigned long long>(), false, claimed.as<uint32_t>()};
        // (a software-pipelined form of the one-window loop — the next unit's keys built and its home group in flight while the current one is
        // probed — needed 75 registers and was slower; it is not kept)
        mark(INSERT_BEGIN);
        ac_launch_occ<AC_INSERT_CTAS>("insert", &stream, ins, (g_end - g_first + 63) / 64 * 32);     // one warp per 64 windows
        mark(INSERT_END);
        ac_d2h(hc, counters.p, sizeof hc, &stream); ac_sync(&stream);
        if (hc[2] && cap != safe_cap) { cap = safe_cap; continue; }         // the estimate was off (it is an estimate): start again with the safe size
        if (hc[2]) throw std::runtime_error("k-mer table overflow");
        if (hc[3] && !big_counts) { big_counts = true; continue; }          // a k-mer with half a million occurrences: counts move to the 32-bit side array
        break;
    }
    ++table_attempt;
    n_dotted = hc[1];
}

// The list of distinct k-mers (their slots) from the claim bits, and with `with_filter` the extension filter over them; returns how
// many there are.
template <int W> uint64_t DevicePipeline::Impl::list_claimed(bool with_filter) {
    const uint64_t n_words = (total + 31) / 32;
    claimed_cnt.ensure((n_words + 1) * 4);
    ac_launch("claimed_count", &stream, ClaimedCountBody{claimed.as<uint32_t>(), n_words, claimed_cnt.as<uint32_t>()}, n_words + 1);
    const uint64_t n = scan(&stream, claimed_cnt.as<uint32_t>(), claimed_cnt.as<uint32_t>(), n_words + 1);
    occ_list.ensure((n + 1) * 4);
    if (with_filter) {
        // two entries per distinct k-mer, 3 bits each: about 4 entries per word, one test in 200 passes by chance (26 MB for BASELINE
        // config 2: L2 resident).  AC_EXT_FILTER_WORDS (test hook) shrinks it, so that nearly every test passes.
        static const uint64_t words_env = getenv("AC_EXT_FILTER_WORDS") ? strtoull(getenv("AC_EXT_FILTER_WORDS"), nullptr, 10) : 0;
        n_fwords = words_env ? words_env : n / 2 + 64;
        ext_filter.ensure(n_fwords * 8);
        ac_memset(ext_filter.p, 0, n_fwords * 8, &stream);
    }
    ac_launch("claimed_list", &stream, ClaimedListBody<W>{claimed.as<uint32_t>(), claimed_cnt.as<uint32_t>(), pos_slot.as<uint32_t>(), occ_list.as<uint32_t>(),
                                                          table_view(), make_kparams(k, W), interior8.as<uint8_t>(), with_filter ? ext_filter.as<uint64_t>() : nullptr, n_fwords}, n_words * 32);
    return n;
}
template <int W> uint64_t DevicePipeline::Impl::count_entries_w() {
    require(Stage::TABLE, "build_local must precede the entry export");
    exp_n = list_claimed<W>(false);        // before any merge: the local table
    exp_valid = true;
    return exp_n;
}
void DevicePipeline::export_entries(void* dst, uint64_t cap_records) {
    Impl& m = *impl; m.make_current();
    if (cap_records < m.exp_n) throw std::runtime_error("entry buffer too small");
    ac_launch("export_scatter", &m.stream, ExportScatterBody{m.table_view(), m.occ_list.as<uint32_t>(), (SlotRec*)dst}, m.exp_n);
    ac_sync(&m.stream);
}

template <int W> void DevicePipeline::Impl::merge_w(const void* dev_ptr, uint64_t n) {
    require(Stage::TABLE, "build_local must precede merge_entries");
    const KParams p = make_kparams(k, W);
    ac_launch("merge", &stream, MergeBody<W>{table_view(), p, (const SlotRec*)dev_ptr, pos_slot.as<uint32_t>(), counters.as<unsigned long long>(), claimed.as<uint32_t>()}, n);
    merged.emplace_back(dev_ptr, n);      // folded in again if the union overflows the table (runs_local_w)
}

// ---- stage 2: adjacency over the (now global) table, unitig occurrences along this rank's sequences ----
template <int W> void DevicePipeline::Impl::runs_local_w() {
    require(Stage::TABLE, "build_local must precede runs_local");
    const KParams p = make_kparams(k, W);
    mark(RUNS_BEGIN);
    if (is_multi) {      // the merges may have tripped the limits too
        unsigned long long hc[AC_N_COUNTERS];
        ac_d2h(hc, counters.p, sizeof hc, &stream); ac_sync(&stream);
        if (hc[2] && cap != safe_cap) {
            // This rank's own k-mers fitted the estimated size, the union with the other ranks' did not.  The safe size counts every rank's
            // windows, so it holds the union: build the own table again at that size and fold the same records in again.  Exported entries
            // do not depend on the table's size, so no rank has to export again (ac_entries_merge's buffers stay valid until this returns).
            cap = safe_cap;
            insert_w<W>();
            const TableView tv = table_view();
            for (const auto& e : merged)
                ac_launch("merge", &stream, MergeBody<W>{tv, p, (const SlotRec*)e.first, pos_slot.as<uint32_t>(), counters.as<unsigned long long>(), claimed.as<uint32_t>()}, e.second);
            ac_d2h(hc, counters.p, sizeof hc, &stream); ac_sync(&stream);
        }
        if (hc[2]) throw std::runtime_error("k-mer table overflow while merging");
        if (hc[3] && !big_counts) throw std::runtime_error("a k-mer occurs more than 524287 times across the ranks: not supported by the multi-GPU exchange");
        n_dotted = hc[1];
    }
    any_dotted = n_dotted != 0;
    const TableView tv = table_view();

    flags8.ensure(cap);
    n_slots_used = list_claimed<W>(true);   // distinct canonical k-mers (with the other ranks' after a merge)
    const AdjacencyBody<W> adj{tv, p, any_dotted, occ_list.as<uint32_t>(), flags8.as<uint8_t>(), ext_filter.as<uint64_t>(), n_fwords};
    if (is_multi && exp_valid && exp_n + 64 < n_slots_used) {      // the merged table holds every rank's k-mers; this rank's own ones were listed (and counted) before the merge
        const uint64_t n_cw = (total + 31) / 32, n_adj = exp_n + 64;
        if (getenv("AC_HOST_PROFILE")) fprintf(stderr, "[device] adjacency flags for this rank's own k-mers: at most %llu of %llu\n", (unsigned long long)n_adj, (unsigned long long)n_slots_used);
        ac_launch("adjacency", &stream, AdjacencyOwnBody<W>{adj, claimed_cnt.as<uint32_t>(), g_begin >> 5, std::min<uint64_t>((g_end + 31) >> 5, n_cw)}, n_adj);
    } else ac_launch("adjacency", &stream, adj, n_slots_used);
    mark(ADJACENCY_END);

    const uint64_t n_bwords = (total + 31) / 32;
    bmask.ensure(n_bwords * sizeof(uint32_t)); bcount.ensure(n_bwords * sizeof(uint32_t)); boff.ensure(n_bwords * sizeof(uint32_t));
    ac_launch("boundaries", &stream, BoundaryBody{packed.as<uint64_t>(), seqs.as<SeqInfo>(), n_seqs, p.h, g_begin, g_end, pos_slot.as<uint32_t>(),
                                                  flags8.as<uint8_t>(), interior8.as<uint8_t>(), bmask.as<uint32_t>(), bcount.as<uint32_t>()}, n_bwords * 32);
    n_runs = scan(&stream, bcount.as<uint32_t>(), boff.as<uint32_t>(), n_bwords);
    mark(BOUNDARIES_END);
    run_start.ensure(n_runs * sizeof(uint64_t)); run_len.ensure(n_runs * 4); run_hs.ensure(n_runs * 4); run_ts.ensure(n_runs * 4);
    ac_launch("run_scatter", &stream, RunScatterBody{bmask.as<uint32_t>(), boff.as<uint32_t>(), run_start.as<uint64_t>()}, n_bwords);
    ac_launch("run_ends", &stream, RunEndsLocalBody{seqs.as<SeqInfo>(), n_seqs, run_start.as<uint64_t>(), n_runs, pos_slot.as<uint32_t>(),
                                                    run_len.as<uint32_t>(), run_hs.as<uint32_t>(), run_ts.as<uint32_t>()}, n_runs);
    n_own_runs = n_runs;
    stage = Stage::RUNS;
}

void DevicePipeline::export_runs(void* dst, uint64_t cap_records) {
    Impl& m = *impl; m.make_current();
    m.require(Stage::RUNS, "runs_local must precede export_runs");
    if (cap_records < m.n_runs) throw std::runtime_error("run buffer too small");
    ac_launch("run_export", &m.stream, RunExportBody{m.run_start.as<uint64_t>(), m.run_len.as<uint32_t>(), m.run_hs.as<uint32_t>(), m.run_ts.as<uint32_t>(),
                                                     m.slots.as<Slot>(), slot_gpos_bits(m.total), (RunRec*)dst}, m.n_runs);
    ac_sync(&m.stream);
}

void DevicePipeline::import_runs(const void* dev_ptr, uint64_t n) {
    Impl& m = *impl; m.make_current();
    m.require(Stage::RUNS, "runs_local must precede import_runs");
    m.n_runs = n;
    m.run_start.ensure(n * sizeof(uint64_t)); m.run_len.ensure(n * 4); m.run_hs.ensure(n * 4); m.run_ts.ensure(n * 4);
    RunImportBody body{(const RunRec*)dev_ptr, m.pos_slot.as<uint32_t>(), m.run_start.as<uint64_t>(), m.run_len.as<uint32_t>(), m.run_hs.as<uint32_t>(), m.run_ts.as<uint32_t>(), 0, {0}, {nullptr}};
    ac_launch("run_import", &m.stream, body, n);
}

void DevicePipeline::import_runs_from(const void* const* ptrs, const uint64_t* counts, uint32_t n_ranks) {
    Impl& m = *impl; m.make_current();
    m.require(Stage::RUNS, "runs_local must precede import_runs");
    if (n_ranks == 0 || n_ranks > AC_MAX_RANKS) throw std::runtime_error("import_runs: bad rank count");
    RunImportBody body{nullptr, m.pos_slot.as<uint32_t>(), nullptr, nullptr, nullptr, nullptr, n_ranks, {0}, {nullptr}};
    for (uint32_t q = 0; q < n_ranks; ++q) { body.first[q + 1] = body.first[q] + counts[q]; body.src[q] = (const RunRec*)ptrs[q]; }
    const uint64_t n = m.n_runs = body.first[n_ranks];
    m.run_start.ensure(n * sizeof(uint64_t)); m.run_len.ensure(n * 4); m.run_hs.ensure(n * 4); m.run_ts.ensure(n * 4);
    body.run_start = m.run_start.as<uint64_t>(); body.run_len = m.run_len.as<uint32_t>(); body.run_hs = m.run_hs.as<uint32_t>(); body.run_ts = m.run_ts.as<uint32_t>();
    ac_launch("run_import", &m.stream, body, n);
}

// ---- stage 3: unitigs, seeds, links, seed order and the host-ready arrays (over every occurrence handed to it) ----
void DevicePipeline::finish(PipelineResult& out, bool keep_positions, bool fused, bool split_paths) {
    Impl& m = *impl; m.make_current(); const int W = m.W;
    if (split_paths && !fused) throw std::runtime_error("split path lines need the fused finish");
    AC_DISPATCH_W(m.unitigs_w, out)
    m.host_arrays();
    m.paths();
    m.work_list();
    // simplify_structure and save_gfa on the device: fused builds only (a plain build hands the host the graph as built)
    if (fused && m.R.n_cands > 0) m.simplify();
    m.mark(SIMPLIFY_END);
    if (fused) {
        m.renumber();
        if (m.U < 100000000u) m.gfa(split_paths);
    }
    m.mark(GFA_END);
    m.results(out, keep_positions, fused);
}

// The part that depends on the key width: run keys, unitigs, their seed k-mers and the links
template <int W> void DevicePipeline::Impl::unitigs_w(PipelineResult& out) {
    require(Stage::RUNS, "runs_local must precede finish");
    const KParams p = make_kparams(k, W);
    const TableView tv = table_view();
    out = PipelineResult();
    out.W = W; out.capacity = cap; out.n_slots_used = n_slots_used; out.n_dotted = n_dotted;
    R = Pending();
    mark(FINISH_BEGIN);
    run_uk.ensure(n_runs * 4); run_dir.ensure(n_runs);
    is_rep.ensure(n_runs * 4); rep_idx.ensure(n_runs * 4); run_unitig.ensure(n_runs * 4);
    uid_rep.ensure(cap * 4); slot_unitig.ensure(cap * 4);
    ac_memset(uid_rep.p, 0xFF, cap * 4, &stream);
    ac_launch("run_key", &stream, RunKeyBody{packed.as<uint64_t>(), p.h, run_start.as<uint64_t>(), run_hs.as<uint32_t>(), run_ts.as<uint32_t>(),
                                             run_uk.as<uint32_t>(), run_dir.as<uint8_t>(), uid_rep.as<uint32_t>()}, n_runs);
    ac_launch("rep_flag", &stream, RepFlagBody{run_uk.as<uint32_t>(), uid_rep.as<uint32_t>(), is_rep.as<uint32_t>()}, n_runs);
    U = scan(&stream, is_rep.as<uint32_t>(), rep_idx.as<uint32_t>(), n_runs);
    unitigs.ensure((size_t)U * sizeof(DeviceUnitig));
    ac_launch("run_assign", &stream, RunAssignBody{run_start.as<uint64_t>(), run_len.as<uint32_t>(), run_uk.as<uint32_t>(), run_dir.as<uint8_t>(),
                                                   uid_rep.as<uint32_t>(), rep_idx.as<uint32_t>(), run_hs.as<uint32_t>(), run_ts.as<uint32_t>(), tv,
                                                   run_unitig.as<uint32_t>(), unitigs.as<DeviceUnitig>(), slot_unitig.as<uint32_t>()}, n_runs);
    mark(UNITIGS_END);

    // ---- seed k-mer / orientation per unitig ----
    nchunks.ensure(((size_t)U + 1) * 4); chunk_off.ensure(((size_t)U + 1) * 4);
    ac_launch("chunk_count", &stream, ChunkCountBody{unitigs.as<DeviceUnitig>(), nchunks.as<uint32_t>()}, U);
    ac_memset(nchunks.as<uint32_t>() + U, 0, 4, &stream);
    n_chunks = scan(&stream, nchunks.as<uint32_t>(), chunk_off.as<uint32_t>(), (uint64_t)U + 1);
    partial.ensure((size_t)n_chunks * sizeof(MinPartial<W>));
    ac_launch("chunk_min", &stream, ChunkMinBody<W>{packed.as<uint64_t>(), seqs.as<SeqInfo>(), n_seqs, p, unitigs.as<DeviceUnitig>(), U,
                                                    chunk_off.as<uint32_t>(), partial.as<MinPartial<W>>()}, n_chunks);
    ac_launch("unitig_min", &stream, UnitigMinBody<W>{chunk_off.as<uint32_t>(), partial.as<MinPartial<W>>(), unitigs.as<DeviceUnitig>()}, U);
    mark(SEEDS_END);

    // ---- links ----
    link_count.ensure((size_t)U * 2 * 4); links.ensure((size_t)U * 2 * AC_MAX_LINKS * 4);
    ac_launch("links", &stream, LinkBody<W>{tv, p, any_dotted, unitigs.as<DeviceUnitig>(), pos_slot.as<uint32_t>(), slot_unitig.as<uint32_t>(),
                                            link_count.as<uint32_t>(), links.as<uint32_t>()}, (uint64_t)U * 2);
    mark(LINKS_END);
}

// Seed order, the host-ready arrays in it, the unitigs' sequences in one arena, and the links as CSR
void DevicePipeline::Impl::host_arrays() {
    // ---- seed order: stable LSD radix sort of the unitigs by their seed k-mer ----
    sort_a.ensure((size_t)U * 4); sort_b.ensure((size_t)U * 4); sort_ra.ensure((size_t)U * sizeof(SortRec)); sort_rb.ensure((size_t)U * sizeof(SortRec));
    const SeedLess seed_less{unitigs.as<DeviceUnitig>(), W};
    const uint32_t* perm = sort_indices(&stream, seed_less, U, sort_a.as<uint32_t>(), sort_b.as<uint32_t>(), sort_ra.as<SortRec>(), sort_rb.as<SortRec>());
    mark(SEED_SORT_END);
    // ---- host-ready arrays in seed order ----
    rank.ensure((size_t)U * 4); d_len.ensure((size_t)U * 4); d_depth.ensure((size_t)U * 4); need.ensure(((size_t)U + 1) * 4);
    d_seq_off.ensure((size_t)U * 8); d_min_fpos.ensure((size_t)U * 4); d_min_rpos.ensure((size_t)U * 4);
    ac_launch("seed_gather", &stream, SeedGatherBody{perm, unitigs.as<DeviceUnitig>(), U, rank.as<uint32_t>(), d_len.as<uint32_t>(), d_depth.as<uint32_t>(),
                                                     need.as<uint32_t>(), d_min_fpos.as<uint32_t>(), d_min_rpos.as<uint32_t>()}, (uint64_t)U + 1);
    // the arena must stay below 4 GB for the 32-bit scan; sum(len) <= windows
    if (n_windows + (uint64_t)U * 2 * AC_SEQ_SLACK >= 0xFFFFFFF0ull) throw std::runtime_error("unitig sequence arena would exceed 4 GB");
    const uint64_t arena_bytes = scan(&stream, need.as<uint32_t>(), need.as<uint32_t>(), (uint64_t)U + 1);
    ac_launch("seq_off", &stream, SeqOffBody{need.as<uint32_t>(), d_seq_off.as<uint64_t>()}, U);
    d_arena.ensure(arena_bytes);
    ac_launch("emit_seq", &stream, EmitSeqBody{packed.as<uint64_t>(), make_kparams(k, W).h, unitigs.as<DeviceUnitig>(), U, chunk_off.as<uint32_t>(), rank.as<uint32_t>(),
                                               d_seq_off.as<uint64_t>(), d_arena.as<char>()}, n_chunks);
    R.arena_final = arena_bytes; R.arena_src = &d_arena;
    // links -> CSR in seed-strand order
    const uint32_t n_strands = 2 * U;
    strand_cnt.ensure(((size_t)n_strands + 1) * 4); d_next_off.ensure(((size_t)n_strands + 1) * 4);
    prev_cnt.ensure(((size_t)n_strands + 1) * 4); d_prev_off.ensure(((size_t)n_strands + 1) * 4);
    ac_launch("link_count", &stream, LinkCountBody{link_count.as<uint32_t>(), rank.as<uint32_t>(), unitigs.as<DeviceUnitig>(), n_strands, strand_cnt.as<uint32_t>()},
              (uint64_t)n_strands + 1);
    const uint64_t n_links = R.n_links = scan(&stream, strand_cnt.as<uint32_t>(), d_next_off.as<uint32_t>(), (uint64_t)n_strands + 1);
    d_next.ensure(n_links * 4); d_prev.ensure(n_links * 4);
    ac_memset(prev_cnt.p, 0, ((size_t)n_strands + 1) * 4, &stream);
    d_small.ensure(64); ac_memset(d_small.p, 0, 64, &stream);           // [0] hairpin links
    ac_launch("link_order", &stream, LinkOrderBody{link_count.as<uint32_t>(), links.as<uint32_t>(), rank.as<uint32_t>(), unitigs.as<DeviceUnitig>(),
                                                   d_next_off.as<uint32_t>(), d_next.as<UStrand>(), prev_cnt.as<uint32_t>(), d_small.as<uint32_t>()}, n_strands);
    scan(&stream, prev_cnt.as<uint32_t>(), d_prev_off.as<uint32_t>(), (uint64_t)n_strands + 1, false);      // the total is n_links again: no read-back, the stream carries on
    ac_memset(prev_cnt.p, 0, ((size_t)n_strands + 1) * 4, &stream);    // reused as the fill cursor
    ac_launch("prev_fill", &stream, PrevFillBody{d_next_off.as<uint32_t>(), d_next.as<UStrand>(), d_prev_off.as<uint32_t>(), prev_cnt.as<uint32_t>(), d_prev.as<UStrand>()}, n_strands);
    ac_launch("prev_sort", &stream, PrevSortBody{d_prev_off.as<uint32_t>(), d_prev.as<UStrand>()}, n_strands);
}

// The path of every sequence, the unitig records the host works on, and their numbering
void DevicePipeline::Impl::paths() {
    d_path.ensure(n_runs * 4); d_path_off.ensure(((size_t)n_seqs + 1) * 8);
    ac_launch("path", &stream, PathBody{seqs.as<SeqInfo>(), n_seqs, run_start.as<uint64_t>(), run_len.as<uint32_t>(), run_unitig.as<uint32_t>(), rank.as<uint32_t>(),
                                        unitigs.as<DeviceUnitig>(), d_path.as<UStrand>(), d_min_fpos.as<uint32_t>(), d_min_rpos.as<uint32_t>()}, n_runs);
    d_rec.ensure((size_t)U * sizeof(UnitigRec));
    ac_launch("pack_rec", &stream, PackRecBody{d_seq_off.as<uint64_t>(), d_len.as<uint32_t>(), d_min_fpos.as<uint32_t>(), d_min_rpos.as<uint32_t>(), d_rec.as<UnitigRec>()}, U);
    ac_launch("path_off", &stream, PathOffBody{seqs.as<SeqInfo>(), n_seqs, run_start.as<uint64_t>(), n_runs, d_path_off.as<uint64_t>()}, (uint64_t)n_seqs + 1);
    // the unitig numbers of the freshly built graph (the rank buffer is free again and holds the 8-base prefixes)
    num_prefix.ensure((size_t)U * 8);
    ac_launch("number_key", &stream, NumberKeyBody{d_rec.as<UnitigRec>(), d_arena.as<char>(), num_prefix.as<uint64_t>()}, U);
    const NumberLess number_less{d_rec.as<UnitigRec>(), d_depth.as<uint32_t>(), d_arena.as<char>(), num_prefix.as<uint64_t>(), nullptr};
    R.order_built = sort_indices(&stream, number_less, U, sort_a.as<uint32_t>(), sort_b.as<uint32_t>(), sort_ra.as<SortRec>(), sort_rb.as<SortRec>());
}

// The work list of expand_repeats, in the numbering order just found
void DevicePipeline::Impl::work_list() {
    d_fixed.ensure((size_t)U * 4); ac_memset(d_fixed.p, 0, (size_t)U * 4, &stream);
    uint8_t* seed_start = d_fixed.as<uint8_t>(); uint8_t* seed_end = seed_start + U; uint8_t* fix_start = R.fix_start = seed_end + U; uint8_t* fix_end = fix_start + U;
    ac_launch("fixed_seed", &stream, FixedSeedBody{d_path_off.as<uint64_t>(), d_path.as<UStrand>(), seed_start, seed_end}, n_seqs);
    ac_copy_dd(fix_start, seed_start, (size_t)U * 2, &stream);
    ac_launch("fixed_spread", &stream, FixedSpreadBody{seed_start, seed_end, d_next_off.as<uint32_t>(), d_next.as<UStrand>(), d_prev_off.as<uint32_t>(), d_prev.as<UStrand>(),
                                                       fix_start, fix_end}, U);
    const CandidateView cview{R.order_built, d_next_off.as<uint32_t>(), d_next.as<UStrand>(), d_prev_off.as<uint32_t>(), d_prev.as<UStrand>(), fix_start, fix_end};
    cand_flag.ensure((2 * (size_t)U + 1) * 4); cand_index.ensure((2 * (size_t)U + 1) * 4);
    ac_launch("candidate_flag", &stream, CandidateFlagBody{cview, U, cand_flag.as<uint32_t>()}, 2ull * U + 1);
    const uint64_t n_cands = R.n_cands = scan(&stream, cand_flag.as<uint32_t>(), cand_index.as<uint32_t>(), 2ull * U + 1);
    d_cands.ensure((n_cands + 1) * sizeof(ExpandCandidate)); d_cand_at.ensure(2 * (size_t)U * 4 + 4); d_deps.ensure((size_t)U * sizeof(ExpandDeps) + 4); d_spec.ensure((n_cands + 1) * 4);
    ac_launch("candidate_fill", &stream, CandidateFillBody{cview, cand_flag.as<uint32_t>(), cand_index.as<uint32_t>(), d_cands.as<ExpandCandidate>(), d_cand_at.as<int32_t>()}, 2ull * U);
    ac_launch("dependents", &stream, DependentsBody{d_next_off.as<uint32_t>(), d_next.as<UStrand>(), d_prev_off.as<uint32_t>(), d_prev.as<UStrand>(), d_cand_at.as<int32_t>(),
                                                    d_deps.as<ExpandDeps>()}, U);
    ac_launch("common_length", &stream, CommonLengthBody{d_cands.as<ExpandCandidate>(), d_rec.as<UnitigRec>(), d_arena.as<char>(), d_spec.as<uint32_t>()}, n_cands);
    mark(WORK_LIST_END);
}

// simplify_structure's repeat expansion: `while expand_repeats() > 0 {}`
void DevicePipeline::Impl::simplify() {
    const uint64_t n_cands = R.n_cands, arena_bytes = R.arena_final;
    d_pred.ensure(n_cands * 7 * 4); d_level.ensure(n_cands * 4); d_flagmax.ensure(32); d_counters64.ensure((AC_PASS_WORDS + 8) * 8);
    d_dirty.ensure(((n_cands + 63) / 64) * 8 + 8); d_exhausted.ensure(n_cands + 8);
    unsigned long long* c64 = d_counters64.as<unsigned long long>();         // SimplifyCoopBody's counters, then its eight result words
    unsigned long long* res = c64 + AC_PASS_WORDS;
    ac_launch("level_pred", &stream, LevelPredBody{d_cands.as<ExpandCandidate>(), d_deps.as<ExpandDeps>(), d_pred.as<int32_t>()}, n_cands);
    ac_memset(d_level.p, 0, n_cands * 4, &stream); ac_memset(d_flagmax.p, 0, 32, &stream);
    ac_launch_coop("levels", &stream, LevelsCoopBody{d_pred.as<int32_t>(), d_level.as<uint32_t>(), d_flagmax.as<uint32_t>(), n_cands}, n_cands, 4096);
    ac_memset(d_counters64.p, 0, (AC_PASS_WORDS + 8) * 8, &stream);
    const RelocBoundBody bound_body{d_cands.as<ExpandCandidate>(), d_rec.as<UnitigRec>(), d_cand_at.as<int32_t>(), c64 + AC_PASS_SET(1) + 1};     // the first pass's bound: into the set it does not use
    ac_launch("reloc_bound", &stream, bound_body, n_cands);
    uint32_t fm[8]; unsigned long long h64[AC_PASS_WORDS + 8];
    ac_d2h(fm, d_flagmax.p, 32, &stream); ac_d2h(h64, c64, sizeof h64, &stream); ac_sync(&stream);
    if (fm[4]) throw std::runtime_error("candidate levels did not settle");
    unsigned long long bound = 0; for (int x = 0; x < AC_BOUND_STRIPES; ++x) bound += h64[AC_PASS_SET(1) + 1 + x];
    if (arena_bytes + bound >= 0xFFFFFFF0ull) throw std::runtime_error("unitig sequence arena would exceed 4 GB");
    // room for the first pass and, usually, for all that follow (each later pass can ask for less than the one before it asked for at most)
    d_arena2.ensure(arena_bytes + 2 * bound + 64);
    ac_copy_dd(d_arena2.p, d_arena.p, arena_bytes, &stream);
    const unsigned long long start = arena_bytes;
    ac_h2d(c64, &start, 8, &stream);
    ac_memset(c64 + AC_PASS_SET(1), 0, AC_PASS_SET_WORDS * 8, &stream);
    ac_memset(d_dirty.p, 0, ((n_cands + 63) / 64) * 8 + 8, &stream); ac_memset(d_exhausted.p, 0, n_cands + 8, &stream);
    // one launch for as many passes as the arena has room for
    static const bool always_grow = getenv("AC_DEVICE_TIGHT_ARENA") != nullptr;   // test hook: one pass per launch, the growth path before every pass
    uint32_t next_set = 0, next_due = 0; uint64_t passes = 0;
    const uint32_t due_stride = fm[3] + 2;
    d_due.ensure((size_t)3 * due_stride * 4); ac_memset(d_due.p, 0, (size_t)3 * due_stride * 4, &stream);
    for (bool first = true;; first = false) {
        const ApplyLevelBody apply{d_cands.as<ExpandCandidate>(), d_deps.as<ExpandDeps>(), d_level.as<uint32_t>(), 0, d_spec.as<uint32_t>(),
                                   d_rec.as<UnitigRec>(), d_arena2.as<char>(), c64, c64, d_dirty.as<uint64_t>(), d_exhausted.as<uint8_t>(), first, c64 + AC_PASS_REMOVED};
        const uint64_t room = always_grow ? 0 : d_arena2.cap;
        ac_launch_coop("simplify", &stream, SimplifyCoopBody{apply, bound_body, n_cands, d_flagmax.as<uint32_t>() + 3, c64, res, room, next_set, first,
                                                             d_due.as<uint32_t>(), due_stride, next_due}, n_cands, 64);
        ac_d2h(h64, c64, sizeof h64, &stream); ac_sync(&stream);
        const unsigned long long* r = h64 + AC_PASS_WORDS;
        R.arena_final = h64[0]; R.bases_removed = h64[AC_PASS_REMOVED]; R.any_moved = r[1] != 0;
        passes += r[2]; next_set = (uint32_t)r[5]; next_due = (uint32_t)r[7];
        if (getenv("AC_HOST_PROFILE")) fprintf(stderr, "[device] expand_repeats launch: %llu passes (%llu so far), %u levels, %llu candidates, %llu left on the work list, last pass moved %llu bases\n",
                                               r[2], (unsigned long long)passes, fm[3], (unsigned long long)n_cands, r[4], r[0]);
        if (r[0] == 0) break;                                                          // the last expand_repeats() call moved nothing
        if (passes > 1000000) throw std::runtime_error("repeat expansion did not settle");
        bound = r[3];                                                                  // the launch stopped for want of room: make it
        if (R.arena_final + bound >= 0xFFFFFFF0ull) throw std::runtime_error("unitig sequence arena would exceed 4 GB");
        d_arena3.ensure(std::max<size_t>((R.arena_final + bound) * 2 + 64, d_arena3.cap + (always_grow ? 64 : 0)));
        ac_copy_dd(d_arena3.p, d_arena2.p, R.arena_final, &stream); ac_sync(&stream);
        std::swap(d_arena2.p, d_arena3.p); std::swap(d_arena2.cap, d_arena3.cap);
    }
    R.arena_src = &d_arena2;
}

// simplify_structure ends with renumber_unitigs (:38): stable with respect to the numbering the passes ran in
void DevicePipeline::Impl::renumber() {
    if (!R.any_moved) { R.final_order = R.order_built; return; }     // nothing moved: the stable sort would change nothing
    d_pos.ensure((size_t)U * 4); sort_c.ensure((size_t)U * 4); sort_d.ensure((size_t)U * 4);
    ac_launch("inverse_perm", &stream, InversePermBody{R.order_built, d_pos.as<uint32_t>()}, U);
    ac_launch("number_key", &stream, NumberKeyBody{d_rec.as<UnitigRec>(), R.arena_src->as<char>(), num_prefix.as<uint64_t>()}, U);
    const NumberLess final_less{d_rec.as<UnitigRec>(), d_depth.as<uint32_t>(), R.arena_src->as<char>(), num_prefix.as<uint64_t>(), d_pos.as<uint32_t>()};
    R.final_order = sort_indices(&stream, final_less, U, sort_c.as<uint32_t>(), sort_d.as<uint32_t>(), sort_ra.as<SortRec>(), sort_rb.as<SortRec>());
}

// save_gfa (unitig_graph.rs:317-360): H, S, L and P lines rendered here.  split_paths: the P lines are printed by the ranks that own the
// sequences (render_path_lines).
void DevicePipeline::Impl::gfa(bool split_paths) {
    d_pos2.ensure((size_t)U * 4);
    ac_launch("inverse_perm", &stream, InversePermBody{R.final_order, d_pos2.as<uint32_t>()}, U);
    const GfaView gv{R.final_order, d_pos2.as<uint32_t>(), d_rec.as<UnitigRec>(), R.arena_src->as<char>(), d_depth.as<uint32_t>(), d_next_off.as<uint32_t>(), d_next.as<UStrand>()};
    gfa_s_size.ensure(((size_t)U + 1) * 4); gfa_l_size.ensure(((size_t)U + 1) * 4); gfa_pieces.ensure(((size_t)U + 1) * 4);
    const uint64_t steps = split_paths ? 0 : n_runs;
    d_last.ensure(steps + 8); gfa_p_size.ensure((steps + 1) * 4);
    ac_launch("gfa_size", &stream, GfaSizeBody{gv, U, gfa_s_size.as<uint32_t>(), gfa_l_size.as<uint32_t>()}, (uint64_t)U + 1);
    ac_launch("gfa_chunk_count", &stream, GfaChunkCountBody{gv, U, gfa_pieces.as<uint32_t>()}, (uint64_t)U + 1);
    // the scans, their totals read back together (one round trip)
    d_totals.ensure(64); ac_memset(d_totals.p, 0, 64, &stream);
    if (!split_paths) {
        ac_memset(d_last.p, 0, steps + 8, &stream);
        ac_launch("path_last", &stream, PathLastBody{d_path_off.as<uint64_t>(), d_last.as<uint8_t>()}, n_seqs);
        ac_launch("path_size", &stream, PathSizeBody{d_path.as<UStrand>(), d_pos2.as<uint32_t>(), d_last.as<uint8_t>(), steps, gfa_p_size.as<uint32_t>()}, steps + 1);
        scan.keep_total(&stream, gfa_p_size.as<uint32_t>(), steps + 1, d_totals.as<uint32_t>() + 3);
    }
    scan.keep_total(&stream, gfa_s_size.as<uint32_t>(), (uint64_t)U + 1, d_totals.as<uint32_t>() + 0);
    scan.keep_total(&stream, gfa_l_size.as<uint32_t>(), (uint64_t)U + 1, d_totals.as<uint32_t>() + 1);
    scan.keep_total(&stream, gfa_pieces.as<uint32_t>(), (uint64_t)U + 1, d_totals.as<uint32_t>() + 2);
    uint32_t tot[4];
    ac_d2h(tot, d_totals.p, 16, &stream); ac_sync(&stream);
    const uint64_t s_bytes = tot[0], l_bytes = tot[1], n_pieces = tot[2], p_list_bytes = tot[3];
    char head[64]; const uint64_t head_bytes = (uint64_t)snprintf(head, sizeof head, "H\tVN:Z:1.0\tKM:i:%u\n", k);
    if (path_wrap_total == 0 && n_seqs) throw std::runtime_error("set_path_line_texts() must precede a build that renders the GFA");
    const uint64_t p_bytes = split_paths ? 0 : p_list_bytes + path_wrap_total;
    R.gfa_bytes = head_bytes + s_bytes + l_bytes + p_bytes;
    d_text.ensure(R.gfa_bytes + 64);
    char* text = d_text.as<char>();
    ac_h2d(text, head, head_bytes, &stream);       // `head` is on the stack: synchronised below before it goes out of scope (h2d from pageable memory is staged by the driver at call time)
    ac_launch("gfa_segment", &stream, GfaSegmentBody{gv, gfa_s_size.as<uint32_t>(), text + head_bytes}, U);
    ac_launch("gfa_sequence", &stream, GfaSequenceBody{gv, U, gfa_pieces.as<uint32_t>(), gfa_s_size.as<uint32_t>(), text + head_bytes}, n_pieces);
    ac_launch("gfa_link", &stream, GfaLinkBody{gv, gfa_l_size.as<uint32_t>(), text + head_bytes + s_bytes}, U);
    const PathLineView pv{d_path_off.as<uint64_t>(), n_seqs, gfa_p_size.as<uint32_t>(), d_wrap_off.as<uint64_t>(), d_pre_len.as<uint32_t>(), d_suf_len.as<uint32_t>(),
                          d_blob.as<char>(), d_blob_off.as<uint64_t>(), 0};
    char* p_text = text + head_bytes + s_bytes + l_bytes;
    if (!split_paths) {
        ac_launch("path_text", &stream, PathTextFullBody{d_path.as<UStrand>(), d_pos2.as<uint32_t>(), d_last.as<uint8_t>(), pv, p_text}, steps);
        ac_launch("path_wrap", &stream, PathWrapBody{pv, p_text}, 2ull * n_seqs);
    }
    R.paths_split = split_paths;
    R.gfa_on_device = true;
}

// ---- results to the host (pinned) ----
void DevicePipeline::Impl::results(PipelineResult& out, bool keep_positions, bool fused) {
    if (before_results && *before_results) (*before_results)();
    out.fused = fused; out.graph_fetched = false;
    if (fused && !R.gfa_on_device) throw std::runtime_error("fused build: the device GFA writer did not run");
    uint64_t d2h = 0;
    if (R.gfa_on_device) {
        h_text.ensure(R.gfa_bytes + 64);
        ac_d2h(h_text.p, d_text.p, R.gfa_bytes, &stream); d2h += R.gfa_bytes;
    }
    uint32_t small[16];
    ac_d2h(small, d_small.p, 64, &stream); ac_sync(&stream); d2h += 64;
    out.links_single = (R.n_links - small[0]) / 2 + small[0];
    out.length_before = n_slots_used;                      // every canonical k-mer lies in exactly one unitig and a trimmed unitig is as long as its chain
    out.length_after = n_slots_used - R.bases_removed;
    out.gfa_text = R.gfa_on_device ? h_text.as<char>() : nullptr; out.gfa_bytes = R.gfa_on_device ? R.gfa_bytes : 0;
    out.n_unitigs = U; out.n_runs = n_runs; out.n_seqs = n_seqs; out.n_links = R.n_links;
    out.h2d_bytes = uploaded_bytes + (uint64_t)n_seqs * sizeof(SeqInfo);
    out.d2h_bytes = d2h;
    if (!fused) pull_graph(out, keep_positions);
    else { mark(ALL_BUT_ARENA); mark(RESULTS_END); arena_pending = true; }
}

// The graph arrays (unitig records, sequences, links, paths, and the numbering and expand_repeats work list of the graph as built, or
// the final numbering after a fused build) into pinned host memory: at once in a plain build, on request after a fused one.
void DevicePipeline::Impl::pull_graph(PipelineResult& out, bool keep_positions) {
    const uint64_t n_links = R.n_links, n_cands = R.n_cands; const uint32_t n_strands = 2 * U;
    const uint64_t arena_cap = R.arena_final + R.arena_final / 4 + (1u << 20);     // head room for relocations during repeat expansion
    h_rec.ensure((size_t)U * sizeof(UnitigRec)); h_depth.ensure((size_t)U * 4);
    h_arena.ensure(arena_cap); h_next_off.ensure(((size_t)n_strands + 1) * 4); h_prev_off.ensure(((size_t)n_strands + 1) * 4);
    h_next.ensure(n_links * 4 + 4); h_prev.ensure(n_links * 4 + 4); h_path.ensure(n_runs * 4 + 4); h_path_off.ensure(((size_t)n_seqs + 1) * 8);
    uint64_t d2h = 0;
    auto pull = [&](PinBuf& dst, DevBuf& src, size_t bytes) { if (bytes) ac_d2h(dst.p, src.p, bytes, &stream); d2h += bytes; };
    pull(h_rec, d_rec, (size_t)U * sizeof(UnitigRec)); pull(h_depth, d_depth, (size_t)U * 4);
    const bool plain = !out.fused;
    if (plain) { h_order.ensure((size_t)U * 4 + 4); if (U) { ac_d2h(h_order.p, R.order_built, (size_t)U * 4, &stream); d2h += (size_t)U * 4; } }
    pull(h_next_off, d_next_off, ((size_t)n_strands + 1) * 4); pull(h_prev_off, d_prev_off, ((size_t)n_strands + 1) * 4);
    pull(h_next, d_next, n_links * 4); pull(h_prev, d_prev, n_links * 4); pull(h_path, d_path, n_runs * 4); pull(h_path_off, d_path_off, ((size_t)n_seqs + 1) * 8);
    if (keep_positions) {
        h_run_start.ensure(n_runs * 8 + 8); h_run_len.ensure(n_runs * 4 + 4);
        pull(h_run_start, run_start, n_runs * 8); pull(h_run_len, run_len, n_runs * 4);
    }
    if (plain) {
        h_cands.ensure((n_cands + 1) * sizeof(ExpandCandidate)); h_deps.ensure((size_t)U * sizeof(ExpandDeps) + 4); h_spec.ensure((n_cands + 1) * 4); h_fixed.ensure((size_t)U * 2 + 4);
        pull(h_cands, d_cands, n_cands * sizeof(ExpandCandidate)); pull(h_deps, d_deps, (size_t)U * sizeof(ExpandDeps)); pull(h_spec, d_spec, n_cands * 4);
        if (U) { ac_d2h(h_fixed.p, R.fix_start, (size_t)U * 2, &stream); d2h += (size_t)U * 2; }
    } else { h_order2.ensure((size_t)U * 4 + 4); if (U) { ac_d2h(h_order2.p, R.final_order, (size_t)U * 4, &stream); d2h += (size_t)U * 4; } }
    // The sequences (most of the bytes) go last: the caller gets the graph structure as soon as everything else has
    // landed and lists the repeat-expansion candidates while the arena is still on its way (complete() waits for it).
    mark(ALL_BUT_ARENA);
    pull(h_arena, *R.arena_src, R.arena_final);
    out.d2h_bytes += d2h;
    mark(RESULTS_END);
    wait_mark(ALL_BUT_ARENA);
    out.graph_fetched = true;
    out.rec = h_rec.as<UnitigRec>(); out.depth = h_depth.as<uint32_t>();
    out.order = plain ? h_order.as<uint32_t>() : nullptr; out.final_order = plain ? nullptr : h_order2.as<uint32_t>();
    out.n_cands = plain ? n_cands : 0; out.cands = plain ? h_cands.as<ExpandCandidate>() : nullptr; out.deps = plain ? h_deps.as<ExpandDeps>() : nullptr;
    out.spec_len = plain ? h_spec.as<uint32_t>() : nullptr;
    out.fixed_start = plain ? h_fixed.as<uint8_t>() : nullptr; out.fixed_end = plain ? h_fixed.as<uint8_t>() + U : nullptr;
    out.arena = h_arena.as<char>(); out.arena_used = R.arena_final; out.arena_cap = arena_cap;
    out.next_off = h_next_off.as<uint32_t>(); out.next = h_next.as<UStrand>(); out.prev_off = h_prev_off.as<uint32_t>(); out.prev = h_prev.as<UStrand>();
    out.path_off = h_path_off.as<uint64_t>(); out.path = h_path.as<UStrand>();
    out.run_start = keep_positions ? h_run_start.as<uint64_t>() : nullptr; out.run_len = keep_positions ? h_run_len.as<uint32_t>() : nullptr;
    arena_pending = true;
}

void DevicePipeline::complete(PipelineResult& out) {
    Impl& m = *impl; m.make_current();
    if (!m.arena_pending) return;
    ac_sync(&m.stream);
    m.arena_pending = false;
    PipelineTimings& t = out.t;
    const struct { float* field; Mark from, to; } spans[] = {
        {&t.h2d, UPLOAD_BEGIN, UPLOAD_END}, {&t.pack, PACK_BEGIN, PACK_END}, {&t.sample, PACK_END, SAMPLE_END}, {&t.insert, SAMPLE_END, TABLE_END},
        {&t.insert_kernel, INSERT_BEGIN, INSERT_END}, {&t.adjacency, RUNS_BEGIN, ADJACENCY_END}, {&t.boundaries, ADJACENCY_END, BOUNDARIES_END},
        {&t.runs, FINISH_BEGIN, UNITIGS_END}, {&t.unitigs, UNITIGS_END, SEEDS_END}, {&t.links, SEEDS_END, LINKS_END}, {&t.seed_sort, LINKS_END, SEED_SORT_END},
        {&t.emit, SEED_SORT_END, WORK_LIST_END}, {&t.simplify, WORK_LIST_END, SIMPLIFY_END}, {&t.gfa, SIMPLIFY_END, GFA_END}, {&t.d2h, GFA_END, RESULTS_END}};
    for (const auto& s : spans) *s.field = m.between(s.from, s.to);
    t.total = m.between(PACK_BEGIN, TABLE_END) + m.between(RUNS_BEGIN, BOUNDARIES_END) + m.between(FINISH_BEGIN, RESULTS_END);
}

// ---- multi-GPU, path lines by owner (DESIGN.md §7): the rank that finished the graph hands every occurrence's final "<number><sign>" to
// the rank that owns the sequence; every rank prints the P lines of its own sequences and copies them out through its own PCIe link ----
void DevicePipeline::export_path_tokens(void* dst, uint64_t stride, const uint64_t* counts, uint32_t n_ranks) {
    Impl& m = *impl; m.make_current();
    if (m.stage < Stage::RUNS || !m.R.gfa_on_device || !m.R.paths_split) throw std::runtime_error("export_path_tokens follows a finish with split path lines");
    if (n_ranks == 0 || n_ranks > AC_MAX_RANKS) throw std::runtime_error("export_path_tokens: bad rank count");
    PathTokenBody body{m.d_path.as<UStrand>(), m.d_pos2.as<uint32_t>(), (uint32_t*)dst, stride, n_ranks, {0}};
    for (uint32_t q = 0; q < n_ranks; ++q) { if (counts[q] > stride) throw std::runtime_error("export_path_tokens: a rank holds more occurrences than the stride"); body.first[q + 1] = body.first[q] + counts[q]; }
    if (body.first[n_ranks] != m.n_runs) throw std::runtime_error("export_path_tokens: the counts do not add up to the occurrences imported");
    ac_launch("path_tokens", &m.stream, body, m.n_runs);
}
void DevicePipeline::render_path_lines(const void* tokens, uint64_t n_tokens, const char** text, uint64_t* bytes) {
    Impl& m = *impl; m.make_current();
    m.require(Stage::RUNS, "runs_local must precede render_path_lines");
    if (n_tokens != m.n_own_runs) throw std::runtime_error("render_path_lines: one token per occurrence of this rank's sequences is expected");
    if (m.path_pre.size() != m.n_seqs) throw std::runtime_error("set_path_line_texts() must precede render_path_lines");
    const uint32_t lo = m.own_seq_lo, hi = m.own_seq_hi, n_own = hi - lo;
    uint64_t wrap_lo = 0, wrap_hi = 0;
    for (uint32_t i = 0; i < hi; ++i) { const uint64_t b = (uint64_t)m.path_pre[i] + m.path_suf[i]; wrap_hi += b; if (i < lo) wrap_lo += b; }
    uint64_t total_bytes = 0;
    if (n_own) {
        const uint64_t steps = n_tokens;
        m.d_own_off.ensure(((size_t)n_own + 1) * 8); m.d_own_last.ensure(steps + 8); m.d_own_size.ensure((steps + 1) * 4);
        // this rank's occurrences are the first n_own_runs entries of run_start (the finishing rank imported its own block first)
        ac_launch("path_off", &m.stream, PathOffBody{m.seqs.as<SeqInfo>() + lo, n_own, m.run_start.as<uint64_t>(), steps, m.d_own_off.as<uint64_t>()}, (uint64_t)n_own + 1);
        ac_memset(m.d_own_last.p, 0, steps + 8, &m.stream);
        ac_launch("path_last", &m.stream, PathLastBody{m.d_own_off.as<uint64_t>(), m.d_own_last.as<uint8_t>()}, n_own);
        ac_launch("path_size", &m.stream, PathSizeBody{(const UStrand*)tokens, nullptr, m.d_own_last.as<uint8_t>(), steps, m.d_own_size.as<uint32_t>()}, steps + 1);
        const uint64_t list_bytes = m.scan(&m.stream, m.d_own_size.as<uint32_t>(), m.d_own_size.as<uint32_t>(), steps + 1);
        total_bytes = list_bytes + (wrap_hi - wrap_lo);
        m.d_ptext.ensure(total_bytes + 64);
        const PathLineView pv{m.d_own_off.as<uint64_t>(), n_own, m.d_own_size.as<uint32_t>(), m.d_wrap_off.as<uint64_t>() + lo, m.d_pre_len.as<uint32_t>() + lo,
                              m.d_suf_len.as<uint32_t>() + lo, m.d_blob.as<char>(), m.d_blob_off.as<uint64_t>() + lo, wrap_lo};
        ac_launch("path_text", &m.stream, PathTextFullBody{(const UStrand*)tokens, nullptr, m.d_own_last.as<uint8_t>(), pv, m.d_ptext.as<char>()}, steps);
        ac_launch("path_wrap", &m.stream, PathWrapBody{pv, m.d_ptext.as<char>()}, 2ull * n_own);
        m.h_ptext.ensure(total_bytes + 64);
        ac_d2h(m.h_ptext.p, m.d_ptext.p, total_bytes, &m.stream);
    }
    ac_sync(&m.stream);
    *text = total_bytes ? m.h_ptext.as<char>() : nullptr; *bytes = total_bytes;
}

void DevicePipeline::build_local(uint32_t seq_lo, uint32_t seq_hi, bool multi) {
    Impl& m = *impl; m.make_current(); const int W = m.W;
    AC_DISPATCH_W(m.local_w, seq_lo, seq_hi, multi)
}
uint64_t DevicePipeline::count_entries() {
    Impl& m = *impl; m.make_current(); const int W = m.W;
    uint64_t count = 0;
    AC_DISPATCH_W(count = m.count_entries_w)
    return count;
}
void DevicePipeline::merge_entries(const void* dev_ptr, uint64_t n) {
    Impl& m = *impl; m.make_current(); const int W = m.W;
    AC_DISPATCH_W(m.merge_w, dev_ptr, n)
}
void DevicePipeline::runs_local() {
    Impl& m = *impl; m.make_current(); const int W = m.W;
    AC_DISPATCH_W(m.runs_local_w)
}
uint64_t DevicePipeline::local_runs() const { return impl->n_runs; }
void DevicePipeline::import_runs_padded(const void* dev_ptr, uint64_t stride, const uint64_t* counts, uint32_t n_ranks) {
    if (n_ranks == 0 || n_ranks > AC_MAX_RANKS) throw std::runtime_error("import_runs_padded: bad rank count");
    const void* ptrs[AC_MAX_RANKS];
    for (uint32_t q = 0; q < n_ranks; ++q) { if (counts[q] > stride) throw std::runtime_error("import_runs_padded: a rank holds more records than the stride"); ptrs[q] = (const char*)dev_ptr + (size_t)q * stride * sizeof(RunRec); }
    import_runs_from(ptrs, counts, n_ranks);
}
const void* DevicePipeline::export_entries_own(uint64_t* n) {
    const uint64_t count = count_entries();
    impl->own_entries.ensure((count + 1) * sizeof(SlotRec));
    export_entries(impl->own_entries.p, count);
    *n = count;
    return impl->own_entries.p;
}
const void* DevicePipeline::export_runs_own(uint64_t* n) {
    Impl& m = *impl; m.make_current();
    m.own_runs.ensure((m.n_runs + 1) * sizeof(RunRec));
    export_runs(m.own_runs.p, m.n_runs);
    *n = m.n_runs;
    return m.own_runs.p;
}
void DevicePipeline::enable_peer_access(const int* devices, int n) {
#ifndef AC_EMULATE
    for (int a = 0; a < n; ++a)
        for (int b = 0; b < n; ++b) {
            if (a == b) continue;
            int can = 0;
            AC_CUDA_CHECK(cudaDeviceCanAccessPeer(&can, devices[a], devices[b]));
            if (!can) throw std::runtime_error("device " + std::to_string(devices[a]) + " cannot map the memory of device " + std::to_string(devices[b]) + " (no peer access)");
            AC_CUDA_CHECK(cudaSetDevice(devices[a]));
            const cudaError_t e = cudaDeviceEnablePeerAccess(devices[b], 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) throw std::runtime_error(std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e));
            cudaGetLastError();
        }
#else
    (void)devices; (void)n;
#endif
}
void* DevicePipeline::strand_block(uint32_t seq_lo, uint32_t seq_hi, uint64_t* n_bytes) {
    Impl& m = *impl;
    if (seq_lo > seq_hi || seq_hi > m.n_seqs || m.total == 0) throw std::runtime_error("strand_block: bad range, or nothing uploaded");
    const SeqInfo* q = m.host_seqs.data();
    const uint64_t b0 = seq_lo < m.n_seqs ? q[seq_lo].start : m.total, b1 = seq_hi < m.n_seqs ? q[seq_hi].start : m.total;
    *n_bytes = b1 - b0;
    return m.ascii.as<uint8_t>() + b0;
}
void DevicePipeline::fetch_graph(PipelineResult& out, bool keep_positions) {
    Impl& m = *impl; m.make_current();
    if (m.stage < Stage::RUNS || !out.fused) throw std::runtime_error("fetch_graph follows a fused build");
    if (out.graph_fetched) return;
    m.pull_graph(out, keep_positions);
}

void DevicePipeline::build(PipelineResult& out, bool keep_positions, bool fused) {   // single GPU: every sequence is local, nothing to exchange
    build_local(0, impl->n_seqs, false);
    runs_local();
    finish(out, keep_positions, fused);
}
