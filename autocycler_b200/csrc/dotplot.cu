// Device part of `autocycler dotplot`: all-vs-all k-mer dots (dotplot.rs:394-450).  This file compiles with nvcc for sm_90a (product)
// and with g++ -DAC_EMULATE (tests/emu, serial execution of the same bodies).
#include "commands.h"

#include <cmath>

#define AC_NONE32 0xFFFFFFFFu
// ------------------------------------------------------------------------------------------------
// dotplot: all-vs-all k-mer dots (dotplot.rs:394-450), see DESIGN.md §14
// ------------------------------------------------------------------------------------------------
// Window j of sequence b matches window p of sequence a forward when a[p..p+k] == b[j..j+k] and in reverse when revcomp(a[p..p+k]) ==
// b[j..j+k] (get_all_kmer_positions, :433-450).  For windows of only ACGT both relations are "same canonical k-mer": forward when the
// two windows have the same orientation, reverse otherwise.  So the dots are the ordered pairs of windows within each group of equal
// canonical keys, and a pixel's colour is the one of its largest dotplot_key (commands.h), whatever order the dots arrive in.
#define AC_DOT_CHUNK 64        // consecutive dots per thread
AC_HD uint32_t dot_base(uint8_t c) { return c == 'A' ? 0u : c == 'C' ? 1u : c == 'G' ? 2u : c == 'T' ? 3u : 4u; }
// (pos as f64 / bp_per_pixel).round() as u32 + start (:401, :405): round half away from zero, Rust's saturating cast (NaN to 0), a
// wrapping u32 add.  The f64 division is IEEE round-to-nearest on the device as on the host, so both get the same pixel.
AC_HD uint32_t dot_px(uint32_t start, uint32_t pos, double bpp) {
    const double v = round((double)pos / bpp);
    return start + (!(v > 0.0) ? 0u : v >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)v);
}

// One thread per window: the window's 2-bit key on both strands (base b of a strand in word b / 32 at bit 2 (b % 32)), the smaller one
// as the canonical key, the orientation, the pixel and the window's tag (dotplot_key with pair = the window's sequence).  A window with
// another byte than ACGT gets rep = NONE: the host matches those (a reverse complement keeps such a byte, so they match nothing else).
template <int W> struct DotWindowBody {
    const uint8_t* bytes; const DotplotSeq* seqs; uint32_t n_seqs, k; double bpp;
    uint64_t* keys; uint32_t* px; uint64_t* tag; uint32_t* rep;
    AC_D void operator()(uint64_t i) const {
        uint32_t lo = 0, hi = n_seqs;               // the last sequence whose first window is <= i (those without windows share the next base)
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (seqs[mid].window_base <= i) lo = mid; else hi = mid; }
        const DotplotSeq s = seqs[lo];
        const uint32_t j = (uint32_t)(i - s.window_base);
        const uint8_t* w = bytes + s.off + j;
        uint64_t f[W], r[W];
        uint32_t bad = 0;
#pragma unroll
        for (int x = 0; x < W; ++x) {
            uint64_t fw = 0, rw = 0;
            const uint32_t b0 = 32u * (uint32_t)x, b1 = k < b0 + 32u ? k : b0 + 32u;
            for (uint32_t b = b0; b < b1; ++b) {
                const uint32_t c = dot_base(w[b]), d = dot_base(w[k - 1 - b]);
                bad |= c >> 2;
                fw |= (uint64_t)(c & 3u) << (2 * (b - b0));
                rw |= (uint64_t)(3u - (d & 3u)) << (2 * (b - b0));
            }
            f[x] = fw; r[x] = rw;
        }
        int cmp = 0;
#pragma unroll
        for (int x = W - 1; x >= 0; --x) if (cmp == 0 && f[x] != r[x]) cmp = f[x] < r[x] ? -1 : 1;
        const bool forward = cmp <= 0;              // a window that is its own reverse complement is forward: at one j the forward hit wins
#pragma unroll
        for (int x = 0; x < W; ++x) keys[i * W + x] = forward ? f[x] : r[x];
        px[i] = dot_px(s.start_px, j, bpp);
        tag[i] = ((uint64_t)lo << 34) | ((uint64_t)j << 2) | ((uint64_t)forward << 1) | 1u;
        rep[i] = bad ? AC_NONE32 : (uint32_t)i;
    }
};

// Open addressing over 8-byte slots: the key's hash in the high half, (window + 1) in the low half, 0 = empty.  A window that finds
// its fingerprint compares the full key with the slot's window before it joins that window's group, so a hash collision never makes
// a dot.  The table has at least twice as many slots as windows and cannot fill.
template <int W> struct DotInsertBody {
    const uint64_t* keys; uint64_t* table; uint64_t mask; uint32_t* rep;
    AC_D void operator()(uint64_t i) const {
        if (rep[i] == AC_NONE32) return;
        uint64_t key[W];
        uint64_t h = 0x243F6A8885A308D3ull;
#pragma unroll
        for (int x = 0; x < W; ++x) { key[x] = keys[i * W + x]; h ^= key[x]; h *= 0x9E3779B97F4A7C15ull; h ^= h >> 32; }
        h ^= h >> 29; h *= 0xBF58476D1CE4E5B9ull; h ^= h >> 32;
        const uint64_t mine = (h & 0xFFFFFFFF00000000ull) | (i + 1);
        for (uint64_t s = h & mask;; s = (s + 1) & mask) {
            uint64_t cur = ac_ld_volatile(table + s);
            if (cur == 0) {
                cur = ac_atomic_cas(table + s, (uint64_t)0, mine);
                if (cur == 0) return;               // i leads its group (rep[i] == i already)
            }
            if ((cur >> 32) == (mine >> 32)) {
                const uint64_t r = (cur & 0xFFFFFFFFull) - 1;
                bool same = true;
#pragma unroll
                for (int x = 0; x < W; ++x) same &= keys[r * W + x] == key[x];
                if (same) { rep[i] = (uint32_t)r; return; }
            }
        }
    }
};

struct DotCountBody {                               // group sizes, at the group's leading window
    const uint32_t* rep; uint32_t* cnt;
    AC_D void operator()(uint64_t i) const { if (rep[i] != AC_NONE32) ac_atomic_add(cnt + rep[i], 1u); }
};
struct DotScatterBody {                             // counting sort by group: pixel and tag of every window, grouped
    const uint32_t* rep; const uint32_t* off; uint32_t* fill; const uint32_t* px; const uint64_t* tag; uint32_t* gpx; uint64_t* gtag;
    AC_D void operator()(uint64_t i) const {
        const uint32_t r = rep[i];
        if (r == AC_NONE32) return;
        const uint32_t p = off[r] + ac_atomic_add(fill + r, 1u);
        gpx[p] = px[i]; gtag[p] = tag[i];
    }
};
struct DotLeadBody {                                // 1 at every group's leading window
    const uint32_t* rep; uint32_t* flag;
    AC_D void operator()(uint64_t i) const { flag[i] = rep[i] == (uint32_t)i ? 1u : 0u; }
};
struct DotGroupBody {                               // group g: where its windows start, how many, and its dots (size squared, u64)
    const uint32_t* rep; const uint32_t* gid; const uint32_t* off; const uint32_t* cnt; uint32_t* gstart; uint32_t* gsize; uint64_t* gdots;
    AC_D void operator()(uint64_t i) const {
        if (rep[i] != (uint32_t)i) return;
        const uint32_t g = gid[i];
        gstart[g] = off[i]; gsize[g] = cnt[i]; gdots[g] = (uint64_t)cnt[i] * cnt[i];
    }
};
// The dots, AC_DOT_CHUNK consecutive ones per thread over the scan of the groups' squared sizes, so that one large group (a
// homopolymer) is spread over as many threads as its dots need.  Dot (u, v) of a group: u is the row window (sequence a, pixel x), v
// the column window (sequence b, window j, pixel y).  The atomic is skipped when the pixel already holds a larger key: pixels on the
// diagonals are hit many times when a pixel spans many bases.
struct DotPairBody {
    const uint64_t* goff; const uint32_t* gstart; const uint32_t* gsize; uint32_t G;
    const uint32_t* gpx; const uint64_t* gtag; uint64_t n_dots; uint32_t n_seqs, res; uint64_t* pix;
    AC_D void operator()(uint64_t t) const {
        uint64_t d = t * AC_DOT_CHUNK;
        const uint64_t end = d + AC_DOT_CHUNK < n_dots ? d + AC_DOT_CHUNK : n_dots;
        uint32_t lo = 0, hi = G;                    // the group holding dot d: the last one that starts at or before it
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (goff[mid] <= d) lo = mid; else hi = mid; }
        uint32_t g = lo, base = gstart[g], s = gsize[g];
        const uint64_t local = d - goff[g];
        uint32_t uu = (uint32_t)(local / s), vv = (uint32_t)(local % s);
        uint32_t xu = gpx[base + uu];
        uint64_t tu = gtag[base + uu], pair_hi = ((tu >> 34) * n_seqs) << 34;
        for (; d < end; ++d) {
            const uint32_t y = gpx[base + vv];
            if (xu < res && y < res) {
                const uint64_t tv = gtag[base + vv];
                const uint64_t key = ((tv & ~2ull) + pair_hi) | (~(tu ^ tv) & 2ull);
                uint64_t* p = pix + (uint64_t)y * res + xu;
                if (*p < key) ac_atomic_max(p, key);
            }
            if (++vv == s) {
                vv = 0;
                if (++uu == s) { uu = 0; if (++g >= G) break; base = gstart[g]; s = gsize[g]; }
                xu = gpx[base + uu]; tu = gtag[base + uu]; pair_hi = ((tu >> 34) * n_seqs) << 34;
            }
        }
    }
};
struct DotMergeBody {                               // the host's dots (windows with other bytes than ACGT) into the same maxima
    const uint64_t* idx; const uint64_t* key; uint64_t* pix;
    AC_D void operator()(uint64_t i) const { ac_atomic_max(pix + idx[i], key[i]); }
};
struct DotComposeBody {                             // a pixel with a dot: mediumblue (forward) or firebrick (reverse), :40-41
    const uint64_t* pix; uint8_t* rgb;
    AC_D void operator()(uint64_t p) const {
        const uint64_t key = pix[p];
        if (!key) return;
        const bool fwd = (key & 2u) != 0;
        rgb[3 * p] = fwd ? 0 : 178; rgb[3 * p + 1] = fwd ? 0 : 34; rgb[3 * p + 2] = fwd ? 205 : 34;
    }
};

template <int W> void DeviceDotplot::windows(uint64_t N, uint32_t n_seqs, uint32_t k, double bpp, uint64_t mask) {
    ac_launch("dot_windows", &ctx.stream, DotWindowBody<W>{d_bytes.as<uint8_t>(), d_seqs.as<DotplotSeq>(), n_seqs, k, bpp, d_keys.as<uint64_t>(),
                                                                d_px.as<uint32_t>(), d_tag.as<uint64_t>(), d_rep.as<uint32_t>()}, N);
    ac_launch("dot_insert", &ctx.stream, DotInsertBody<W>{d_keys.as<uint64_t>(), d_table.as<uint64_t>(), mask, d_rep.as<uint32_t>()}, N);
}

void DeviceDotplot::dotplot(const uint8_t* bytes, uint64_t n_bytes, const DotplotSeq* seqs, uint32_t n_seqs, uint32_t k, double bpp, uint32_t res,
                            const uint64_t* host_idx, const uint64_t* host_key, uint64_t n_host, uint8_t* rgb, DotplotRun* run) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    if (k < 1 || k > 128) throw std::runtime_error("dotplot: k must be 1..128");
    if (n_seqs == 0 || n_seqs > AC_DOTPLOT_MAX_SEQS) throw std::runtime_error("dotplot: 1 to 32768 sequences");
    uint64_t N = 0;
    for (uint32_t s = 0; s < n_seqs; ++s) {
        const uint64_t nw = seqs[s].len >= k ? seqs[s].len - k + 1 : 0;
        if (seqs[s].window_base != N || seqs[s].off + seqs[s].len > n_bytes) throw std::runtime_error("dotplot: bad sequence layout");
        N += nw;
    }
    if (N >= 0xFFFFFFFFull) throw std::runtime_error("dotplot: too many windows");
    const int W = (int)((2 * k + 63) / 64);
    const uint64_t P = (uint64_t)res * res;
    DotplotRun r; r.windows = N;
    d_bytes.ensure(n_bytes + 8); d_seqs.ensure((size_t)n_seqs * sizeof(DotplotSeq));
    d_pix.ensure(P * 8); d_rgb.ensure(P * 3);
    if (n_bytes) ac_h2d(d_bytes.p, bytes, n_bytes, st);
    ac_h2d(d_seqs.p, seqs, (size_t)n_seqs * sizeof(DotplotSeq), st);
    ac_h2d(d_rgb.p, rgb, P * 3, st);
    ac_memset(d_pix.p, 0, P * 8, st);
    if (n_host) {
        d_hidx.ensure(n_host * 8); d_hkey.ensure(n_host * 8);
        ac_h2d(d_hidx.p, host_idx, n_host * 8, st); ac_h2d(d_hkey.p, host_key, n_host * 8, st);
    }
    AcTimer timer(st);
    if (N) {
        uint64_t cap = 64;
        while (cap < 2 * N) cap <<= 1;
        d_keys.ensure(N * W * 8); d_px.ensure(N * 4); d_tag.ensure(N * 8); d_rep.ensure(N * 4); d_cnt.ensure(N * 4 + 4);
        d_off.ensure(N * 4 + 4); d_fill.ensure(N * 4 + 4); d_gpx.ensure(N * 4); d_gtag.ensure(N * 8); d_table.ensure(cap * 8);
        ac_memset(d_table.p, 0, cap * 8, st);
        ac_memset(d_cnt.p, 0, N * 4, st); ac_memset(d_fill.p, 0, N * 4, st);
        switch (W) {
            case 1: windows<1>(N, n_seqs, k, bpp, cap - 1); break;
            case 2: windows<2>(N, n_seqs, k, bpp, cap - 1); break;
            case 3: windows<3>(N, n_seqs, k, bpp, cap - 1); break;
            default: windows<4>(N, n_seqs, k, bpp, cap - 1); break;
        }
        uint32_t* rep = d_rep.as<uint32_t>();
        uint32_t* cnt = d_cnt.as<uint32_t>();
        uint32_t* off = d_off.as<uint32_t>();
        ac_launch("dot_count", st, DotCountBody{rep, cnt}, N);
        scan(st, cnt, off, N, false);
        ac_launch("dot_scatter", st, DotScatterBody{rep, off, d_fill.as<uint32_t>(), d_px.as<uint32_t>(), d_tag.as<uint64_t>(),
                                                    d_gpx.as<uint32_t>(), d_gtag.as<uint64_t>()}, N);
        uint32_t* flag = d_fill.as<uint32_t>();          // the fill counts are spent: the leading-window flags, then their ranks
        ac_launch("dot_lead", st, DotLeadBody{rep, flag}, N);
        const uint32_t G = scan(st, flag, flag, N);
        r.groups = G;
        if (G) {
            d_gstart.ensure((size_t)G * 4); d_gsize.ensure((size_t)G * 4); d_gdots.ensure(((size_t)G + 1) * 8);
            uint64_t* gdots = d_gdots.as<uint64_t>();
            ac_memset(gdots + G, 0, 8, st);
            ac_launch("dot_group", st, DotGroupBody{rep, flag, off, cnt, d_gstart.as<uint32_t>(), d_gsize.as<uint32_t>(), gdots}, N);
            scan_u64.run(st, gdots, gdots, (uint64_t)G + 1, false);
            uint64_t D = 0;
            ac_d2h(&D, gdots + G, 8, st); ac_sync(st);
            r.dots = D;
            ac_launch("dot_pairs", st, DotPairBody{gdots, d_gstart.as<uint32_t>(), d_gsize.as<uint32_t>(), G, d_gpx.as<uint32_t>(),
                                                   d_gtag.as<uint64_t>(), D, n_seqs, res, d_pix.as<uint64_t>()},
                      (D + AC_DOT_CHUNK - 1) / AC_DOT_CHUNK);
        }
    }
    if (n_host) ac_launch("dot_merge", st, DotMergeBody{d_hidx.as<uint64_t>(), d_hkey.as<uint64_t>(), d_pix.as<uint64_t>()}, n_host);
    ac_launch("dot_compose", st, DotComposeBody{d_pix.as<uint64_t>(), d_rgb.as<uint8_t>()}, P);
    timer.stop();
    ac_d2h(rgb, d_rgb.p, P * 3, st);
    ac_sync(st);
    r.kernel_ms = timer.ms();
    if (run) *run = r;
}

