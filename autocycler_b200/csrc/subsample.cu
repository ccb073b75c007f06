// Device part of `autocycler subsample` (subsample.rs): the FASTQ record scan, the read statistics and the split into subsets.  This
// file compiles with nvcc for sm_90a (product) and with g++ -DAC_EMULATE (tests/emu, serial execution of the same bodies).
#include "commands.h"

#include <chrono>
#include <utility>

#define AC_NONE32 0xFFFFFFFFu
// ------------------------------------------------------------------------------------------------
// subsample: record scan, statistics and subsets, see DESIGN.md §16
// ------------------------------------------------------------------------------------------------
// Pass 1, one window: a newline mask per 64-byte word and its popcount, the scan of the counts gives every newline's line number, the
// line ends are scattered, and one thread per four lines checks a record and writes its spans and sequence length.
struct SubNewlineBody {                             // word w: bit b of mask[w] set when byte 64w + b is '\n'
    const uint64_t* words; uint64_t* mask; uint32_t* cnt;
    AC_D void operator()(uint64_t w) const {
        uint64_t m = 0;
        for (int x = 0; x < 8; ++x) {
            const uint64_t v = words[8 * w + x];
            for (int b = 0; b < 8; ++b) m |= (uint64_t)(((v >> (8 * b)) & 0xFFu) == '\n') << (8 * x + b);
        }
        mask[w] = m;
        cnt[w] = ac_popc((uint32_t)m) + ac_popc((uint32_t)(m >> 32));
    }
};
struct SubLineEndBody {                             // line_end[line] = the offset of its '\n'
    const uint64_t* mask; const uint32_t* off; uint64_t* line_end;
    AC_D void operator()(uint64_t w) const {
        uint64_t m = mask[w];
        for (uint32_t j = off[w]; m; m &= m - 1, ++j) {
            const uint32_t lo = (uint32_t)m;
            const int b = lo ? ac_ctz(lo) : 32 + ac_ctz((uint32_t)(m >> 32));
            line_end[j] = 64 * w + (uint64_t)b;
        }
    }
};
// Record r holds lines 4r..4r+3 (lines_total of them in the window; the last record of a file may have fewer).  A trailing '\r' is
// stripped from the header, sequence and quality (seq_io's trim_cr); the '+' line's text is dropped.  Checks in order: '@', '+', all
// four lines present, sequence and quality of one length, lengths below 2^32.
struct SubRecordBody {
    const uint8_t* bytes; const uint64_t* line_end; uint64_t lines_total, first; SubRecord* rec; uint32_t* len; uint64_t* bad;
    AC_D void operator()(uint64_t r) const {
        const uint64_t a = 4 * r, have = lines_total - a < 4 ? lines_total - a : 4;
        uint64_t s[4] = {0, 0, 0, 0}, e[4] = {0, 0, 0, 0};
        for (uint64_t k = 0; k < have; ++k) {
            s[k] = a + k == 0 ? 0 : line_end[a + k - 1] + 1;
            e[k] = line_end[a + k];
            if (k != 2 && e[k] > s[k] && bytes[e[k] - 1] == '\r') --e[k];
        }
        uint32_t why = 0;
        if (e[0] == s[0] || bytes[s[0]] != '@') why = SUB_NO_AT;
        else if (have >= 3 && (line_end[a + 2] == s[2] || bytes[s[2]] != '+')) why = SUB_NO_PLUS;
        else if (have < 4) why = SUB_TRUNCATED;
        else if (e[1] - s[1] != e[3] - s[3]) why = SUB_UNEQUAL;
        else if (e[1] - s[1] > 0xFFFFFFFFull || e[0] - s[0] - 1 > 0xFFFFFFFFull) why = SUB_TOO_LONG;
        if (why) { ac_atomic_min(bad, ((first + r) << 3) | why); return; }
        SubRecord o;
        o.head = s[0] + 1; o.head_len = (uint32_t)(e[0] - s[0] - 1);
        o.seq = s[1]; o.seq_len = (uint32_t)(e[1] - s[1]);
        o.qual = s[3];
        rec[r] = o;
        if (len) len[first + r] = o.seq_len;
    }
};

// Statistics without a sort.  Row 0 is the input (rank null); with ranks, row i is subset i.  The ascending n50 is the smallest length
// L with sum(len <= L) >= bases / 2: level 1 sums the lengths by their high 16 bits, the scan of the rows finds the bucket where each
// row's running sum crosses half its bases, and level 2 sums that bucket's lengths by their low 16 bits.
struct SubRow { uint64_t bases, need; uint32_t cross, zeros, n50, pad; };
AC_HD bool sub_member(const uint32_t* rank, uint64_t r, uint64_t n, uint64_t start, uint64_t rps) {
    const uint64_t k = rank[r];
    return (k >= start ? k - start : k + n - start) < rps;
}
struct SubRankBody {
    const uint32_t* order; uint32_t* rank;
    AC_D void operator()(uint64_t p) const { rank[order[p]] = (uint32_t)p; }
};
struct SubHist1Body {
    const uint32_t* len; const uint32_t* rank; uint64_t n; const uint64_t* starts; uint32_t rows; uint64_t rps; uint64_t* h1; SubRow* row;
    AC_D void operator()(uint64_t r) const {
        const uint32_t L = len[r];
        for (uint32_t i = 0; i < rows; ++i) {
            if (rank && !sub_member(rank, r, n, starts[i], rps)) continue;
            if (L) ac_atomic_add(h1 + ((uint64_t)i << 16) + (L >> 16), (uint64_t)L);
            else ac_atomic_add(&row[i].zeros, 1u);
        }
    }
};
struct SubFind1Body {                               // bucket x of the level-1 rows: the row's bases, and its crossing bucket
    const uint64_t* h1; const uint64_t* s1; SubRow* row;
    AC_D void operator()(uint64_t x) const {
        const uint64_t i = x >> 16, base = s1[i << 16], bases = s1[(i + 1) << 16] - base, target = bases / 2;
        if ((x & 0xFFFF) == 0) row[i].bases = bases;
        if (target == 0) return;
        const uint64_t before = s1[x] - base;
        if (before < target && before + h1[x] >= target) { row[i].cross = (uint32_t)(x & 0xFFFF); row[i].need = target - before; }
    }
};
struct SubHist2Body {
    const uint32_t* len; const uint32_t* rank; uint64_t n; const uint64_t* starts; uint32_t rows; uint64_t rps; const SubRow* row; uint64_t* h2;
    AC_D void operator()(uint64_t r) const {
        const uint32_t L = len[r];
        for (uint32_t i = 0; i < rows; ++i) {
            if (row[i].cross != (L >> 16) || (rank && !sub_member(rank, r, n, starts[i], rps))) continue;
            ac_atomic_add(h2 + ((uint64_t)i << 16) + (L & 0xFFFF), (uint64_t)L);
        }
    }
};
struct SubFind2Body {
    const uint64_t* h2; const uint64_t* s2; SubRow* row;
    AC_D void operator()(uint64_t x) const {
        const uint64_t i = x >> 16;
        if (row[i].cross == AC_NONE32) return;
        const uint64_t before = s2[x] - s2[i << 16];
        if (before < row[i].need && before + h2[x] >= row[i].need) row[i].n50 = (row[i].cross << 16) | (uint32_t)(x & 0xFFFF);
    }
};

// Pass 2, one window and one subset: each member record's normalised size, their offsets (a u64 scan), and one warp per record copies
// `@head\nseq\n+\nqual\n` to its offset.
struct SubPickBody {
    const SubRecord* rec; const uint32_t* rank; uint64_t first, n, start, rps; uint64_t* size;
    AC_D void operator()(uint64_t r) const {
        const SubRecord o = rec[r];
        size[r] = sub_member(rank, first + r, n, start, rps) ? (uint64_t)o.head_len + 2 * (uint64_t)o.seq_len + 6 : 0;
    }
};
struct SubGatherBody {
    const uint8_t* bytes; const SubRecord* rec; const uint64_t* off; uint8_t* out;
    AC_D void operator()(uint64_t t) const {
        const uint64_t r = t >> 5, size = off[r + 1] - off[r];
        if (!size) return;
        const SubRecord o = rec[r];
        const uint64_t h = o.head_len, s = o.seq_len;
        uint8_t* dst = out + off[r];
        for (uint64_t k = t & 31; k < size; k += 32) {
            uint8_t c;
            if (k == 0) c = '@';
            else if (k <= h) c = bytes[o.head + k - 1];
            else if (k == h + 1 || k == h + s + 2 || k == h + s + 4 || k == size - 1) c = '\n';
            else if (k <= h + s + 1) c = bytes[o.seq + k - h - 2];
            else if (k == h + s + 3) c = '+';
            else c = bytes[o.qual + k - h - s - 5];
            dst[k] = c;
        }
    }
};

namespace {
double host_ms_since(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}
}  // namespace

SubScan DeviceSubsample::scan_window(const uint8_t* bytes, uint64_t n, bool eof, uint64_t first, bool keep_lengths) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    SubScan out;
    const uint64_t nw = (n + 63) / 64;
    d_bytes.ensure(nw * 64 + 64);
    d_mask.ensure(nw * 8 + 8); d_cnt.ensure(nw * 4 + 4); d_bad.ensure(8);
    const auto t0 = std::chrono::steady_clock::now();
    if (n) ac_h2d(d_bytes.p, bytes, n, st);
    ac_memset(d_bytes.as<uint8_t>() + n, 0, nw * 64 + 64 - n, st);             // no '\n' past the window, and a byte after its end
    ac_memset(d_bad.p, 0xFF, 8, st);
    ac_sync(st);
    copy_ms += host_ms_since(t0);
    AcTimer timer(st);
    ac_launch("sub_newline", st, SubNewlineBody{d_bytes.as<uint64_t>(), d_mask.as<uint64_t>(), d_cnt.as<uint32_t>()}, nw);
    const uint64_t nl = nw ? scan(st, d_cnt.as<uint32_t>(), d_cnt.as<uint32_t>(), nw) : 0;
    const bool tail = eof && n && bytes[n - 1] != '\n';                          // a last line without its newline ends at n
    const uint64_t lines = nl + (tail ? 1 : 0);
    d_line.ensure(lines * 8 + 8);
    uint64_t* line_end = d_line.as<uint64_t>();
    ac_launch("sub_line_end", st, SubLineEndBody{d_mask.as<uint64_t>(), d_cnt.as<uint32_t>(), line_end}, nw);
    if (tail) ac_h2d(line_end + nl, &n, 8, st);
    const uint64_t R = eof ? (lines + 3) / 4 : nl / 4;
    if (R) {
        if (first + R >= 0xFFFFFFFFull) throw std::length_error("subsample: 2^32 - 1 reads or more");
        d_rec.ensure(R * sizeof(SubRecord));
        if (keep_lengths && (first + R) * 4 > d_len.cap) {                     // the file-wide lengths grow, keeping what they hold
            d_len_tmp.ensure(2 * (first + R) * 4);
            if (first) ac_copy_dd(d_len_tmp.p, d_len.p, first * 4, st);
            std::swap(d_len.p, d_len_tmp.p); std::swap(d_len.cap, d_len_tmp.cap);
        }
        ac_launch("sub_record", st, SubRecordBody{d_bytes.as<uint8_t>(), line_end, lines, first, d_rec.as<SubRecord>(),
                                                  keep_lengths ? d_len.as<uint32_t>() : nullptr, d_bad.as<uint64_t>()}, R);
        ac_d2h(&out.bad, d_bad.p, 8, st);
        if (eof) out.cut = n;
        else { ac_d2h(&out.cut, line_end + 4 * R - 1, 8, st); }
    } else if (eof) out.cut = n;
    timer.stop();
    ac_sync(st);
    if (R && !eof) out.cut += 1;
    kernel_ms += timer.ms();
    out.records = R;
    win_records = R; win_bytes = n;
    return out;
}

void DeviceSubsample::rows(uint64_t n, const uint64_t* starts, uint32_t count, uint64_t rps, SubStats* out) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    const bool subsets = starts != nullptr;
    const uint32_t R = subsets ? count : 1;
    const uint64_t cells = (uint64_t)R << 16;
    d_h1.ensure((cells + 1) * 8); d_s1.ensure((cells + 1) * 8); d_h2.ensure((cells + 1) * 8); d_s2.ensure((cells + 1) * 8);
    d_row.ensure(R * sizeof(SubRow));
    if (subsets) { d_starts.ensure(R * 8); ac_h2d(d_starts.p, starts, R * 8, st); }
    ac_memset(d_h1.p, 0, (cells + 1) * 8, st); ac_memset(d_h2.p, 0, (cells + 1) * 8, st);
    std::vector<SubRow> init(R, SubRow{0, 0, AC_NONE32, 0, 0, 0});
    ac_h2d(d_row.p, init.data(), R * sizeof(SubRow), st);
    const uint32_t* rank = subsets ? d_rank.as<uint32_t>() : nullptr;
    const uint64_t* dst = subsets ? d_starts.as<uint64_t>() : nullptr;
    SubRow* row = d_row.as<SubRow>();
    AcTimer timer(st);
    ac_launch("sub_hist1", st, SubHist1Body{d_len.as<uint32_t>(), rank, n, dst, R, rps, d_h1.as<uint64_t>(), row}, n);
    scan_u64.run(st, d_h1.as<uint64_t>(), d_s1.as<uint64_t>(), cells + 1, false);
    ac_launch("sub_find1", st, SubFind1Body{d_h1.as<uint64_t>(), d_s1.as<uint64_t>(), row}, cells);
    ac_launch("sub_hist2", st, SubHist2Body{d_len.as<uint32_t>(), rank, n, dst, R, rps, row, d_h2.as<uint64_t>()}, n);
    scan_u64.run(st, d_h2.as<uint64_t>(), d_s2.as<uint64_t>(), cells + 1, false);
    ac_launch("sub_find2", st, SubFind2Body{d_h2.as<uint64_t>(), d_s2.as<uint64_t>(), row}, cells);
    timer.stop();
    ac_d2h(init.data(), row, R * sizeof(SubRow), st);
    ac_sync(st);
    kernel_ms += timer.ms();
    for (uint32_t i = 0; i < R; ++i) {
        const SubRow& w = init[i];
        out[i].count = subsets ? rps : n;
        out[i].bases = w.bases;
        // half the bases is 0 (every length 0, or one read of length 1 among them): the first length in ascending order
        out[i].n50 = w.bases / 2 ? w.n50 : (w.zeros || w.bases == 0 ? 0 : 1);
    }
}

SubStats DeviceSubsample::input_stats(uint64_t n) { SubStats s; rows(n, nullptr, 1, 0, &s); return s; }

void DeviceSubsample::set_order(const uint32_t* order, uint64_t n) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    d_rank.ensure(n * 4 + 4); d_size.ensure(n * 4 + 4);
    uint32_t* d_order = d_size.as<uint32_t>();                 // the size buffer is free until gather()
    ac_h2d(d_order, order, n * 4, st);
    AcTimer timer(st);
    ac_launch("sub_rank", st, SubRankBody{d_order, d_rank.as<uint32_t>()}, n);
    timer.stop();
    ac_sync(st);
    kernel_ms += timer.ms();
}

void DeviceSubsample::subset_stats(uint64_t n, const uint64_t* starts, uint32_t count, uint64_t rps, SubStats* out) { rows(n, starts, count, rps, out); }

uint64_t DeviceSubsample::gather(uint64_t first, uint64_t n, uint64_t start, uint64_t rps, uint8_t* host_out) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    const uint64_t R = win_records;
    if (!R) return 0;
    d_size.ensure((R + 1) * 8); d_out.ensure(win_bytes + 1);
    uint64_t* size = d_size.as<uint64_t>();
    ac_memset(size + R, 0, 8, st);
    AcTimer timer(st);
    ac_launch("sub_pick", st, SubPickBody{d_rec.as<SubRecord>(), d_rank.as<uint32_t>(), first, n, start, rps, size}, R);
    const uint64_t total = scan_u64.run(st, size, size, R + 1, true);
    ac_launch("sub_gather", st, SubGatherBody{d_bytes.as<uint8_t>(), d_rec.as<SubRecord>(), size, d_out.as<uint8_t>()}, R * 32);
    timer.stop();
    const auto t0 = std::chrono::steady_clock::now();
    if (total) ac_d2h(host_out, d_out.p, total, st);
    ac_sync(st);
    copy_ms += host_ms_since(t0);
    kernel_ms += timer.ms();
    return total;
}
