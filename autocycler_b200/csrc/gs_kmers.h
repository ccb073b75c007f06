// The packed k-mer stream's word helpers, shared by `helper genome_size` (genome_size.cu) and `depth` (depth.cu): a word's 2-bit codes
// and validity mask, the windows that end in it, and the 64-bit mix of a canonical key (DESIGN.md §18, §19).  Device code only.
#pragma once
#include "commands.h"

// Word w of a sequence of len bytes at s: its codes (when code is not null) and its validity mask.
AC_D uint32_t gs_pack_word(const uint8_t* s, uint64_t len, uint64_t w, uint64_t* code) {
    uint64_t c = 0;
    uint32_t v = 0;
    const uint64_t lo = 32 * w, n = len > lo ? (len - lo < 32 ? len - lo : 32) : 0;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t b = s[lo + i] & 0xDFu;                  // uppercase; only a/c/g/t become A/C/G/T
        if (b == 'A' || b == 'C' || b == 'G' || b == 'T') {
            c |= (uint64_t)(((b >> 1) ^ (b >> 2)) & 3u) << (2 * i);
            v |= 1u << i;
        }
    }
    if (code) *code = c;
    return v;
}
// Bit i of the result is set when the k bases ending at base i of word w are all valid (pv: word w-1's mask, 0 before the stream).
AC_HD uint32_t gs_window_ends(uint32_t v, uint32_t pv, uint32_t k) {
    uint64_t a = ((uint64_t)v << 32) | pv;
    for (uint32_t have = 1; have < k;) {                       // runs of `have` set bits -> runs of 2 have (or k) set bits
        const uint32_t s = have < k - have ? have : k - have;
        a &= a << s;
        have += s;
    }
    return (uint32_t)(a >> 32);
}
// 64-bit finalizer (MurmurHash3's fmix64) of a canonical key: the partition is its high product with P, the home slot the high product
// of the remaining fraction with the table's slots.
AC_HD uint64_t gs_mix(uint64_t x) {
    x ^= x >> 33; x *= 0xFF51AFD7ED558CCDull;
    x ^= x >> 33; x *= 0xC4CEB9FE1A85EC53ull;
    return x ^ (x >> 33);
}
