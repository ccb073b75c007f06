// K-mer key arithmetic shared by every kernel (host + device inline functions).
//
// A k-mer over the reference's 5-letter alphabet ['.', 'A', 'C', 'G', 'T'] (kmer_graph.rs:23) is held as
//   * W = ceil(2k/64) 64-bit words of 2-bit base codes (A=0 C=1 G=2 T=3, '.' stored as 0), first base most
//     significant, right-aligned in the W*64-bit integer (w[0] is the most significant word);
//   * d: 0 for a pure ACGT k-mer, +p for p leading dots, -s for s trailing dots.  Dots only ever form a
//     prefix or a suffix run of at most k/2 (sequence.rs:44-46 pads k/2 dots at both ends; end repair,
//     compress.rs:202-236, can only shorten the runs), never both in one k-mer because L >= k.
// Byte order of the reference's keys (kmer_graph.rs:168-173, '.' < 'A' < 'C' < 'G' < 'T') is reproduced by
// key_less5(): (leading dots desc, codes asc, trailing dots desc).
#pragma once
#include "backend.h"

template <int W> struct Key {
    uint64_t w[W];
    int32_t d;
};

struct KParams {
    uint32_t k, h;        // k-mer size, k/2
    uint32_t top_bits;    // valid bits in w[0]: 2k - 64*(W-1)
    uint64_t top_mask;
};

static inline KParams make_kparams(uint32_t k, int W) {
    KParams p; p.k = k; p.h = k / 2; p.top_bits = 2 * k - 64 * (uint32_t)(W - 1);
    p.top_mask = p.top_bits == 64 ? ~0ull : ((1ull << p.top_bits) - 1);
    return p;
}

// One padded input sequence in the global coordinate system (all padded forward strands concatenated).
struct SeqInfo {
    uint64_t start;       // global coordinate of padded byte 0
    uint32_t len;         // L: original contig length == number of k-mer windows
    uint16_t lead, trail; // dots left at the start / end after end repair (0..k/2)
    uint16_t id;          // Sequence.id (position.rs: 15 bits)
    uint16_t pad;
};

AC_HD uint8_t base_code(uint8_t c) { return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : 0; }

template <int W> AC_HD bool key_eq(const Key<W>& a, const Key<W>& b) {
    bool eq = a.d == b.d;
#pragma unroll
    for (int j = 0; j < W; ++j) eq = eq && (a.w[j] == b.w[j]);
    return eq;
}

template <int W> AC_HD int key_cmp_codes(const Key<W>& a, const Key<W>& b) {
#pragma unroll
    for (int j = 0; j < W; ++j) { if (a.w[j] != b.w[j]) return a.w[j] < b.w[j] ? -1 : 1; }
    return 0;
}

// Lexicographic order of the k ASCII bytes with '.' < 'A' < 'C' < 'G' < 'T'.
template <int W> AC_HD bool key_less5(const Key<W>& a, const Key<W>& b) {
    int la = a.d > 0 ? a.d : 0, lb = b.d > 0 ? b.d : 0;
    if (la != lb) return la > lb;
    int c = key_cmp_codes(a, b);
    if (c != 0) return c < 0;
    int ta = a.d < 0 ? -a.d : 0, tb = b.d < 0 ? -b.d : 0;
    return ta > tb;
}

// (key << 2 | code) & mask : drop the first base, append `code` on the right.
template <int W> AC_HD void key_push_right(Key<W>& key, uint64_t code, const KParams& p) {
#pragma unroll
    for (int j = 0; j < W - 1; ++j) key.w[j] = (key.w[j] << 2) | (key.w[j + 1] >> 62);
    key.w[W - 1] = (key.w[W - 1] << 2) | code;
    key.w[0] &= p.top_mask;
}

// (key >> 2) | code << 2(k-1) : drop the last base, prepend `code` on the left.
template <int W> AC_HD void key_push_left(Key<W>& key, uint64_t code, const KParams& p) {
#pragma unroll
    for (int j = W - 1; j > 0; --j) key.w[j] = (key.w[j] >> 2) | (key.w[j - 1] << 62);
    key.w[0] = (key.w[0] >> 2) | (code << (p.top_bits - 2));
}

// `c ? a : b` by value, word by word.  The same choice between two references takes their addresses, and the device compiler then
// keeps both keys in local memory.
template <int W> AC_HD Key<W> key_select(bool c, const Key<W>& a, const Key<W>& b) {
    Key<W> r;
#pragma unroll
    for (int j = 0; j < W; ++j) r.w[j] = c ? a.w[j] : b.w[j];
    r.d = c ? a.d : b.d;
    return r;
}

// The two (k-1)-mers of a k-mer, right-aligned like a key and without dots (a dot at the dropped end goes with it): its first k-1
// bases (the last one dropped) and its last k-1 bases (the first one dropped).
template <int W> AC_HD Key<W> key_prefix(const Key<W>& key) {
    Key<W> r;
#pragma unroll
    for (int j = W - 1; j > 0; --j) r.w[j] = (key.w[j] >> 2) | (key.w[j - 1] << 62);
    r.w[0] = key.w[0] >> 2;
    r.d = 0;
    return r;
}
template <int W> AC_HD Key<W> key_suffix(const Key<W>& key, const KParams& p) {
    Key<W> r = key;
    r.w[0] &= p.top_mask >> 2;
    r.d = 0;
    return r;
}

// code of base at index i (0 = first base).
template <int W> AC_HD uint32_t key_base(const Key<W>& key, uint32_t i, const KParams& p) {
    const uint32_t bit = 2 * (p.k - 1 - i), word = W - 1 - (bit >> 6);
    uint64_t v = 0;
#pragma unroll
    for (int j = 0; j < W; ++j) v = (word == (uint32_t)j) ? key.w[j] : v;     // no dynamic indexing: keeps the key in registers
    return (uint32_t)(v >> (bit & 63)) & 3u;
}

// The centre base is never a dot; the strand whose centre base is A or C is the stored ("canonical")
// one.  k is odd, so a k-mer never equals its own reverse complement.
template <int W> AC_HD bool key_is_canonical(const Key<W>& key, const KParams& p) { return key_base(key, p.h, p) < 2; }

AC_HD uint64_t rev2_64(uint64_t x) {   // reverse the order of the 32 2-bit groups
#ifdef __CUDA_ARCH__
    x = __brevll(x);                                                                  // all 64 bits reversed: the groups are in place, their two bits swapped
    return ((x >> 1) & 0x5555555555555555ull) | ((x & 0x5555555555555555ull) << 1);
#endif
    x = ((x >> 2) & 0x3333333333333333ull) | ((x & 0x3333333333333333ull) << 2);
    x = ((x >> 4) & 0x0F0F0F0F0F0F0F0Full) | ((x & 0x0F0F0F0F0F0F0F0Full) << 4);
    x = ((x >> 8) & 0x00FF00FF00FF00FFull) | ((x & 0x00FF00FF00FF00FFull) << 8);
    x = ((x >> 16) & 0x0000FFFF0000FFFFull) | ((x & 0x0000FFFF0000FFFFull) << 16);
    return (x >> 32) | (x << 32);
}

// Reverse complement (misc.rs:324-342): bases complemented and reversed, '.' stays '.'.
template <int W> AC_HD Key<W> key_rc(const Key<W>& key, const KParams& p) {
    Key<W> r;
    uint64_t t[W];
#pragma unroll
    for (int j = 0; j < W; ++j) t[j] = rev2_64(key.w[W - 1 - j]);   // codes now left-aligned
    const uint32_t sh = 64 - p.top_bits;                             // 0..62
#pragma unroll
    for (int j = W - 1; j >= 0; --j) {
        uint64_t v = t[j] >> sh;
        if (sh && j > 0) v |= t[j - 1] << (64 - sh);
        r.w[j] = ~v;
    }
    r.w[0] &= p.top_mask;
    r.d = -key.d;
    if (key.d != 0) {   // rare: dot positions must hold code 0 again
        uint32_t nd = (uint32_t)(key.d > 0 ? key.d : -key.d);
        for (uint32_t i = 0; i < nd; ++i) {
            uint32_t idx = key.d > 0 ? (p.k - 1 - i) : i;     // old leading dots become trailing and vice versa
            const uint32_t bit = 2 * (p.k - 1 - idx), word = W - 1 - (bit >> 6);
            const uint64_t keep = ~(3ull << (bit & 63));
#pragma unroll
            for (int j = 0; j < W; ++j) r.w[j] &= (word == (uint32_t)j) ? keep : ~0ull;
        }
    }
    return r;
}

// One multiply-add per key word, then two multiply-xorshift rounds.  The slot index takes the top bits (umulhi), the fingerprint the
// low ones.
template <int W> AC_HD uint64_t key_hash(const Key<W>& key) {
    uint64_t h = key.w[0];
#pragma unroll
    for (int j = 1; j < W; ++j) h = h * 0x9E3779B97F4A7C15ull + key.w[j];
    if (key.d != 0) h ^= (uint64_t)(int64_t)key.d * 0xD6E8FEB86659FD93ull;
    h ^= h >> 32; h *= 0xFF51AFD7ED558CCDull;
    h ^= h >> 29; h *= 0xC4CEB9FE1A85EC53ull;
    h ^= h >> 32;
    return h;
}

// 2-bit packed sequence store: base j of the global coordinate system sits in word j>>5 at bits
// [62 - 2*(j&31), 64 - 2*(j&31)), i.e. the words read as one big-endian base stream.  The buffer carries
// W+1 words of zero padding at the end so that fetches never run off it.
// y[0..W) = the 64W bits that start at bit `sh` (0..62, even) of the big-endian bit stream x[0], x[1], ..., x[W].  On the device: the
// stream as 32-bit words, a one-word step when sh >= 32 and one funnel shift per output word (a 64-bit shift pair costs four times that).
template <int W> AC_HD void ac_stream_window(const uint64_t (&x)[W + 1], uint32_t sh, uint64_t (&y)[W]) {
#ifdef __CUDA_ARCH__
    uint32_t z[2 * W + 1];
    const bool step = sh >= 32u;
#pragma unroll
    for (int i = 0; i <= 2 * W; ++i) {
        const uint32_t a = (i & 1) ? (uint32_t)x[i >> 1] : (uint32_t)(x[i >> 1] >> 32);                  // 32-bit word i of the stream
        const uint32_t b = ((i + 1) & 1) ? (uint32_t)x[(i + 1) >> 1] : (uint32_t)(x[(i + 1) >> 1] >> 32);  // word i + 1 (i = 2W: the low half of x[W])
        z[i] = step ? b : a;
    }
#pragma unroll
    for (int j = 0; j < W; ++j) {
        const uint32_t hi = __funnelshift_l(z[2 * j + 1], z[2 * j], sh), lo = __funnelshift_l(z[2 * j + 2], z[2 * j + 1], sh);   // the shift count is taken modulo 32
        y[j] = ((uint64_t)hi << 32) | lo;
    }
#else
#pragma unroll
    for (int j = 0; j < W; ++j) y[j] = sh ? (x[j] << sh) | (x[j + 1] >> (64 - sh)) : x[j];
#endif
}

template <int W> AC_HD Key<W> fetch_codes(const uint64_t* __restrict__ packed, uint64_t gpos, const KParams& p) {
    const uint64_t i0 = gpos >> 5;
    const uint32_t o = 2 * (uint32_t)(gpos & 31);
    uint64_t x[W + 1], y[W];
#pragma unroll
    for (int j = 0; j <= W; ++j) x[j] = packed[i0 + j];
    ac_stream_window<W>(x, o, y);
    Key<W> r;
    const uint32_t sh = 64 - p.top_bits;
#pragma unroll
    for (int j = W - 1; j >= 0; --j) {
        uint64_t v = y[j] >> sh;
        if (sh && j > 0) v |= y[j - 1] << (64 - sh);
        r.w[j] = v;
    }
    r.d = 0;
    return r;
}

AC_HD uint32_t packed_base(const uint64_t* __restrict__ packed, uint64_t g) {
    return (uint32_t)(packed[g >> 5] >> (62 - 2 * (uint32_t)(g & 31))) & 3u;
}

// number of dots in the window starting at padded offset fs of sequence s: +leading / -trailing / 0
AC_HD int32_t window_dots(const SeqInfo& s, uint64_t fs, uint32_t k) {
    if (fs < s.lead) return (int32_t)(s.lead - fs);
    uint64_t limit = (uint64_t)s.len + (k - 1) - s.trail;   // first padded offset that is a trailing dot
    uint64_t end = fs + k;
    return end > limit ? -(int32_t)(end - limit) : 0;
}

// largest i with seqs[i].start <= g
AC_HD uint32_t find_seq(const SeqInfo* __restrict__ seqs, uint32_t n, uint64_t g) {
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (seqs[mid].start <= g) lo = mid; else hi = mid; }
    return lo;
}

// ---- table slot: ONE 64-bit word [ gpos:GB | dotted:1 | fingerprint:33-GB | count:20 | flags:10 ] --------------------------
// gpos   a pointer to one occurrence of the k-mer, like Kmer.pointer (kmer_graph.rs:26-33): keys never live in the table, equality is
//        decided by fetching that occurrence from the packed sequence store (L2 resident).  GB = the bits the input's coordinates
//        need (26 for BASELINE config 2, at most 32); what it leaves goes to the fingerprint (7 bits for config 2), which spares most
//        probes the fetch of an occurrence that turns out to be another k-mer.
// count  Kmer::depth() (kmer_graph.rs:52-55), occurrences on both strands, 20 bits.  Occurrences are added with fire-and-forget
//        atomics (nobody waits for the old value); an adder whose LOADED copy of the slot already shows 2^19 or more raises the count
//        alarm and the build is repeated with the counts in a side array (`count_big`, 32 bits per slot).  The loaded copy lags the
//        true count by at most the adds in flight — fewer than the 270,336 threads an H100 holds — so a count cannot pass from 2^19 to
//        the wrap at 2^20 (524,288 more adds) without some adder loading a value of at least 2^19 on the way: the alarm is exact.
// flags  bit0 first(canonical) bit1 first(rc(canonical)) (kmer_graph.rs:57-60); bits 2..5: base b follows this k-mer somewhere in the
//        input, bits 6..9: base b precedes it (canonical orientation; a lower bound on the node-centric degrees)
// Eight bytes per slot, four slots per 32-byte sector; the table of BASELINE config 2 is about 100 MB.
typedef uint64_t Slot;
#define AC_EMPTY_SLOT (~0ull)                 // gpos all ones is never a window start: GB is chosen so that total <= 2^GB - 1
#define AC_SLOT_COUNT_SHIFT 10
#define AC_SLOT_COUNT_BITS 20
#define AC_SLOT_COUNT_ONE (1ull << AC_SLOT_COUNT_SHIFT)
#define AC_SLOT_COUNT_ALARM (1u << (AC_SLOT_COUNT_BITS - 1))
#define AC_SLOT_FLAG_MASK 0x3FFull
#define AC_SLOT_TAG_SHIFT (AC_SLOT_COUNT_SHIFT + AC_SLOT_COUNT_BITS)
#define AC_SLOT_TAG_BITS(gb) (64u - AC_SLOT_TAG_SHIFT - (gb))
AC_HD uint32_t slot_gpos_bits(uint64_t total) { uint32_t gb = 8; while (gb < 32 && (total >> gb) != 0) ++gb; return gb; }
AC_HD uint64_t slot_gpos(Slot s, uint32_t gb) { return s >> (64 - gb); }
AC_HD uint32_t slot_tag_word(Slot s) {          // bits 30..61 of the slot: the tag in its low bits, the low end of the occurrence pointer above it
#ifdef __CUDA_ARCH__
    return __funnelshift_r((uint32_t)s, (uint32_t)(s >> 32), AC_SLOT_TAG_SHIFT);
#else
    return (uint32_t)(s >> AC_SLOT_TAG_SHIFT);
#endif
}
AC_HD uint32_t slot_tag(Slot s, uint32_t gb) { return (uint32_t)(s >> AC_SLOT_TAG_SHIFT) & ((1u << AC_SLOT_TAG_BITS(gb)) - 1u); }      // dotted bit + fingerprint
AC_HD bool slot_dotted(Slot s, uint32_t gb) { return (s >> (63 - gb)) & 1; }
AC_HD uint32_t slot_count(Slot s) { return (uint32_t)(s >> AC_SLOT_COUNT_SHIFT) & ((1u << AC_SLOT_COUNT_BITS) - 1u); }
AC_HD uint32_t slot_flags(Slot s) { return (uint32_t)s & 0x3FFu; }
AC_HD uint32_t make_tag(bool dotted, uint64_t hash, uint32_t gb) { const uint32_t fb = AC_SLOT_TAG_BITS(gb) - 1u; return ((uint32_t)dotted << fb) | ((uint32_t)hash & ((1u << fb) - 1u)); }
AC_HD Slot make_slot(uint64_t gpos, uint32_t tag, uint32_t count, uint32_t flags, uint32_t gb) {
    return (gpos << (64 - gb)) | ((uint64_t)tag << AC_SLOT_TAG_SHIFT) | ((uint64_t)count << AC_SLOT_COUNT_SHIFT) | flags;
}
AC_HD Slot slot_with_gpos(Slot s, uint64_t gpos, uint32_t gb) { return (s & ((1ull << (64 - gb)) - 1ull)) | (gpos << (64 - gb)); }
#define AC_AUX_FIRST_CANON 1u
#define AC_AUX_FIRST_RC 2u
#define AC_AUX_OBS_OUT_SHIFT 2
#define AC_AUX_OBS_IN_SHIFT 6
// flags8[slot], written by the adjacency kernel: bit0 outOK = outdeg == 1 && !first(rc K), bit1 inOK = indeg == 1 && !first(K) (canonical orientation)
#define AC_FLAG8_OUT_OK 1u
#define AC_FLAG8_IN_OK 2u
// What one rank tells the others about a k-mer of its local table (multi-GPU exchange, "k-mer buckets"): the slot word and the full count.
struct SlotRec { uint64_t slot; uint32_t count; uint32_t pad; };
