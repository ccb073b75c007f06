// `autocycler subsample` on the host (see host_subsample.h).  Citations are file:line in the reference's src/.
#include "host_subsample.h"

#include <sys/stat.h>
#include <zlib.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <stdexcept>

#include "host_cluster.h"
#include "host_io.h"

namespace {
double ms_since(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

uint64_t as_u64(double x) {            // Rust's saturating `f64 as u64` of round() (half away from zero)
    x = std::round(x);
    if (!(x > 0)) return 0;
    if (x >= 18446744073709551616.0) return UINT64_MAX;
    return (uint64_t)x;
}

// rand_chacha 0.9 ChaCha12Rng (the 64-bit block counter from 0, stream 0) seeded by rand_core 0.9's seed_from_u64 (PCG32 steps, one
// u32 of the key per step).  next() returns the keystream's u32 words in order.
struct ChaChaWords {
    uint32_t key[8], buf[16]; uint64_t block = 0; int pos = 16, rounds;
    ChaChaWords(uint64_t state, int rounds) : rounds(rounds) {
        for (int i = 0; i < 8; ++i) {
            state = state * 6364136223846793005ull + 11634580027462260723ull;
            const uint32_t xorshifted = (uint32_t)(((state >> 18) ^ state) >> 27), rot = (uint32_t)(state >> 59);
            key[i] = (xorshifted >> rot) | (xorshifted << ((32 - rot) & 31));
        }
    }
    static uint32_t rotl(uint32_t v, int c) { return (v << c) | (v >> (32 - c)); }
    void refill() {
        const uint32_t in[16] = {0x61707865u, 0x3320646Eu, 0x79622D32u, 0x6B206574u, key[0], key[1], key[2], key[3], key[4], key[5], key[6],
                                 key[7], (uint32_t)block, (uint32_t)(block >> 32), 0, 0};
        uint32_t x[16];
        memcpy(x, in, sizeof x);
        auto qr = [&](int a, int b, int c, int d) {
            x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 16); x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 12);
            x[a] += x[b]; x[d] = rotl(x[d] ^ x[a], 8);  x[c] += x[d]; x[b] = rotl(x[b] ^ x[c], 7);
        };
        for (int r = 0; r < rounds; r += 2) {
            qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15);
            qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14);
        }
        for (int i = 0; i < 16; ++i) buf[i] = x[i] + in[i];
        ++block; pos = 0;
    }
    uint32_t next() { if (pos == 16) refill(); return buf[pos++]; }
};
// rand 0.9 random_range(..bound) on u32: a widening multiply; when the low half exceeds bound.wrapping_neg(), one more word's high half
// is added to the low half and a carry bumps the result.
uint32_t below(ChaChaWords& rng, uint32_t bound) {
    if (bound == 0) return rng.next();
    const uint64_t m = (uint64_t)rng.next() * bound;
    uint32_t hi = (uint32_t)(m >> 32);
    const uint32_t lo = (uint32_t)m;
    if (lo > (uint32_t)(0u - bound)) {
        const uint32_t new_hi = (uint32_t)(((uint64_t)rng.next() * bound) >> 32);
        if ((uint64_t)lo + new_hi > 0xFFFFFFFFull) ++hi;
    }
    return hi;
}

void grow_keep(PinBuf& b, size_t want, size_t keep) {    // pinned memory that keeps its first `keep` bytes
    if (want <= b.cap) return;
    PinBuf nb;
    nb.ensure(want);
    if (keep) memcpy(nb.p, b.p, keep);
    std::swap(b.p, nb.p); std::swap(b.cap, nb.cap);
}
const char* reason_text(uint64_t why) {
    switch (why) {
        case SUB_NO_AT: return "expected '@' at the start of the header line";
        case SUB_NO_PLUS: return "expected '+' at the start of the separator line";
        case SUB_TRUNCATED: return "truncated record";
        case SUB_UNEQUAL: return "sequence and quality lengths differ";
        default: return "a read of 2^32 bases or more";
    }
}

}  // namespace

// str::parse::<f64> (already lowercased): [+-]? then inf, infinity, nan, or digits with an optional '.' and exponent; nothing else, so
// no hex floats and no partial parses.  The value is strtod's, correctly rounded as Rust's is.
bool rust_f64(const std::string& s, double& v) {
    size_t i = 0;
    if (i < s.size() && (s[i] == '+' || s[i] == '-')) ++i;
    const std::string rest = s.substr(i);
    if (rest == "inf" || rest == "infinity" || rest == "nan") {
        v = rest == "nan" ? NAN : (s[0] == '-' ? -INFINITY : INFINITY);
        return true;
    }
    size_t digits = 0;
    while (i < s.size() && isdigit((unsigned char)s[i])) { ++i; ++digits; }
    if (i < s.size() && s[i] == '.') { ++i; while (i < s.size() && isdigit((unsigned char)s[i])) { ++i; ++digits; } }
    if (digits == 0) return false;
    if (i < s.size() && s[i] == 'e') {
        ++i;
        if (i < s.size() && (s[i] == '+' || s[i] == '-')) ++i;
        size_t e = 0;
        while (i < s.size() && isdigit((unsigned char)s[i])) { ++i; ++e; }
        if (e == 0) return false;
    }
    if (i != s.size()) return false;
    v = strtod(s.c_str(), nullptr);
    return true;
}
FastqStream::FastqStream(const std::string& p) : path(p) {
    f = fopen(p.c_str(), "rb");
    if (!f) throw AcIoError{"cannot read " + p};
    unsigned char magic[2] = {0, 0};
    const size_t got = fread(magic, 1, 2, f);
    if (got == 2 && magic[0] == 0x1f && magic[1] == 0x8b) {
        fclose(f); f = nullptr;
        g = gzopen(p.c_str(), "rb");
        if (!g) throw AcIoError{"cannot read " + p};
        gzbuffer(g, 1 << 20);
    } else rewind(f);
}
FastqStream::~FastqStream() { if (f) fclose(f); if (g) gzclose(g); }
size_t FastqStream::read(uint8_t* dst, size_t n) {
    if (f) {
        const size_t got = fread(dst, 1, n, f);
        if (got < n && ferror(f)) throw AcIoError{"cannot read " + path};
        return got;
    }
    const int got = gzread(g, dst, (unsigned)std::min<size_t>(n, 1u << 30));
    if (got < 0) throw InputError{"Error reading FASTQ file: " + path + " is not a valid gzip file"};
    return (size_t)got;
}

void fastq_windows(DeviceSubsample& dev, const std::string& path, uint64_t& window, bool keep_lengths, SubsampleRun& run,
                   const std::function<void(uint64_t, uint64_t)>& each_window) {
    FastqStream in(path);
    struct stat st;
    const uint64_t file_size = in.f && stat(path.c_str(), &st) == 0 ? (uint64_t)st.st_size : 0;
    uint64_t have = 0, first = 0, scanned = 0;
    bool eof = false;
    while (true) {
        const auto t0 = std::chrono::steady_clock::now();
        while (have < window && !eof) {
            if (have == dev.h_win.cap) {
                const uint64_t want = in.f ? std::min<uint64_t>(window, file_size + 64) : std::min<uint64_t>(window, std::max<uint64_t>(2 * dev.h_win.cap, 1 << 20));
                grow_keep(dev.h_win, std::max<uint64_t>(want, have + 1), have);
            }
            const size_t got = in.read(dev.h_win.as<uint8_t>() + have, std::min<uint64_t>(window, dev.h_win.cap) - have);
            if (got == 0) eof = true;
            have += got;
        }
        run.read_ms += ms_since(t0);
        if (eof && have == 0 && scanned) break;                     // the last window ended the file exactly
        ++scanned;
        const SubScan s = dev.scan_window(dev.h_win.as<uint8_t>(), have, eof, first, keep_lengths);
        if (s.bad != AC_SUB_NONE64) {
            const uint64_t why = s.bad & 7;
            const std::string msg = "Error reading FASTQ file: record " + std::to_string((s.bad >> 3) + 1) + ": " + reason_text(why);
            if (why == SUB_TOO_LONG) throw std::length_error(msg);
            throw InputError{msg};
        }
        if (!s.records && !eof) { window *= 2; continue; }        // a record longer than the window: the window grows
        if (keep_lengths) { ++run.windows; run.bytes_scanned += s.cut; }
        each_window(first, s.records);
        first += s.records;
        memmove(dev.h_win.p, dev.h_win.as<uint8_t>() + s.cut, have - s.cut);
        have -= s.cut;
        if (eof) break;
    }
}

uint64_t parse_genome_size(const std::string& text) {
    size_t a = 0, b = text.size();
    while (a < b && isspace((unsigned char)text[a])) ++a;
    while (b > a && isspace((unsigned char)text[b - 1])) --b;
    std::string s = text.substr(a, b - a);
    for (char& c : s) c = (char)tolower((unsigned char)c);
    double v;
    if (rust_f64(s, v)) return as_u64(v);
    const char last = s.empty() ? 0 : s.back();
    const double mult = last == 'k' ? 1e3 : last == 'm' ? 1e6 : last == 'g' ? 1e9 : 0;
    if (mult == 0 || !rust_f64(s.substr(0, s.size() - 1), v)) throw InputError{"cannot interpret genome size"};
    return as_u64(v * mult);
}

std::vector<uint32_t> subsample_rng_words(uint64_t seed, uint64_t n, int rounds) {
    ChaChaWords rng(seed, rounds);
    std::vector<uint32_t> w(n);
    for (uint32_t& x : w) x = rng.next();
    return w;
}

std::vector<uint32_t> subsample_shuffle(uint64_t n, uint64_t seed) {
    std::vector<uint32_t> order(n);
    for (uint64_t i = 0; i < n; ++i) order[i] = (uint32_t)i;
    if (n <= 1) return order;
    ChaChaWords rng(seed, 12);
    // IncreasingUniform::new(rng, 0): chunk is a draw below (m)(m+1)...(m+remaining-1), handed out one index at a time
    uint32_t cn = 0, chunk = 0, remaining = 1;
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t next_n = cn + 1;
        uint32_t next_remaining;
        if (remaining == 0) {
            uint64_t product = next_n, current = next_n + 1;      // calculate_bound_u32
            while (product * current <= 0xFFFFFFFFull) { product *= current; ++current; }
            chunk = below(rng, (uint32_t)product);
            next_remaining = (uint32_t)(current - next_n) - 1;
        } else next_remaining = remaining - 1;
        uint32_t index;
        if (next_remaining == 0) index = chunk;
        else { index = chunk % next_n; chunk /= next_n; }
        remaining = next_remaining; cn = next_n;
        std::swap(order[i], order[index]);
    }
    return order;
}

uint64_t subsample_window_size() {
    const char* e = getenv("AC_SUBSAMPLE_WINDOW");
    if (e && *e) { const unsigned long long w = strtoull(e, nullptr, 10); if (w > 0) return w; }
    return 1ull << 30;
}

void subsample_run(DeviceSubsample& dev, const std::string& reads, const std::string& out_dir, uint64_t genome_size, uint64_t count,
                   double min_depth, uint64_t seed, uint64_t window, bool verbose, SubsampleRun& run) {
    run = SubsampleRun();
    run.genome_size = genome_size;
    dev.kernel_ms = 0.f; dev.copy_ms = 0.0;
    // pass 1 (input_fastq_stats, :103-118): every record checked and its length kept on the device
    uint64_t n = 0;
    fastq_windows(dev, reads, window, true, run, [&](uint64_t, uint64_t r) { n += r; });
    const bool one_window = run.windows == 1;
    run.input = dev.input_stats(n);
    if (verbose) fprintf(stderr, "Input FASTQ:\n  Read count: %llu\n  Read bases: %llu\n  Read N50 length: %llu bp\n\n", (unsigned long long)n,
                         (unsigned long long)run.input.bases, (unsigned long long)run.input.n50);
    // calculate_subsets (:120-144)
    const double total_depth = (double)run.input.bases / (double)genome_size;
    if (verbose) fprintf(stderr, "\nCalculating subset size\n    Autocycler will now calculate the number of reads to put in each subset.\n\n"
                                 "Total read depth: %.1f\xC3\x97\nMean read length: %llu bp\n\n", total_depth,
                         (unsigned long long)as_u64((double)run.input.bases / (double)n));
    if (total_depth < min_depth) throw InputError{"input reads are too shallow to subset"};
    const double subset_depth = min_depth * std::log2(4.0 * total_depth / min_depth) / 2.0;
    const uint64_t rps = as_u64(subset_depth / total_depth * (double)n);
    run.reads_per_subset = rps;
    if (verbose) fprintf(stderr, "Calculating subset sizes:\n  subset_depth = %s * log_2(4 * total_depth / %s) / 2\n               = %.1fx\n"
                                 "  reads per subset: %llu\n\n", format_float(min_depth).c_str(), format_float(min_depth).c_str(), subset_depth,
                         (unsigned long long)rps);
    // save_subsets (:147-167): the shuffle on the host, the membership and every subset's statistics on the device
    if (verbose) fprintf(stderr, "\nSubsetting reads\n    The reads are now shuffled and grouped into subset files.\n\n");
    auto t0 = std::chrono::steady_clock::now();
    const std::vector<uint32_t> order = subsample_shuffle(n, seed);
    run.shuffle_ms = ms_since(t0);
    if (n) dev.set_order(order.data(), n);
    std::vector<uint64_t> starts(count);
    for (uint64_t i = 0; i < count; ++i) starts[i] = as_u64((double)(i * n) / (double)count);
    std::vector<SubStats> outs(count);
    for (uint64_t i = 0; i < count && n; i += 64) {              // 64 histogram rows at a time
        const uint32_t batch = (uint32_t)std::min<uint64_t>(64, count - i);
        dev.subset_stats(n, starts.data() + i, batch, rps, outs.data() + i);
    }
    std::vector<std::string> names(count);
    std::vector<FILE*> files(count, nullptr);
    struct Closer { std::vector<FILE*>& f; ~Closer() { for (FILE* x : f) if (x) fclose(x); } } closer{files};
    for (uint64_t i = 0; i < count; ++i) {
        char num[32];
        snprintf(num, sizeof num, "%02llu", (unsigned long long)(i + 1));
        names[i] = out_dir + "/sample_" + num + ".fastq";
        if (verbose) {
            const uint64_t s = starts[i], e = s + rps;
            if (e > n) fprintf(stderr, "subset %llu:\n  reads %llu-%llu and 1-%llu\n", (unsigned long long)(i + 1), (unsigned long long)(s + 1),
                               (unsigned long long)n, (unsigned long long)(e - n));
            else fprintf(stderr, "subset %llu:\n  reads %llu-%llu\n", (unsigned long long)(i + 1), (unsigned long long)(s + 1), (unsigned long long)e);
            fprintf(stderr, "  %s\n\n", names[i].c_str());
        }
        files[i] = fopen(names[i].c_str(), "wb");
        if (!files[i]) throw AcIoError{"cannot write " + names[i]};
    }
    // pass 2 (write_subsampled_reads, :199-225): the window of pass 1 when there was one, else the file again
    auto write_window = [&](uint64_t first, uint64_t) {
        dev.h_out.ensure(std::max<uint64_t>(dev.h_win.cap, 1) + 1);
        for (uint64_t i = 0; i < count; ++i) {
            const uint64_t bytes = dev.gather(first, n, starts[i], rps, dev.h_out.as<uint8_t>());
            const auto t1 = std::chrono::steady_clock::now();
            if (bytes && fwrite(dev.h_out.p, 1, bytes, files[i]) != bytes) throw AcIoError{"cannot write " + names[i]};
            run.write_ms += ms_since(t1);
        }
    };
    if (n && one_window) write_window(0, n);
    else if (n) fastq_windows(dev, reads, window, false, run, write_window);
    t0 = std::chrono::steady_clock::now();
    for (uint64_t i = 0; i < count; ++i) {
        const bool good = fclose(files[i]) == 0;
        files[i] = nullptr;
        if (!good) throw AcIoError{"cannot write " + names[i]};
    }
    // SubsampleMetrics (metrics.rs:25-42) as serde_yaml 0.9 writes it
    std::string yaml = "input_read_count: " + std::to_string(n) + "\ninput_read_bases: " + std::to_string(run.input.bases) +
                       "\ninput_read_n50: " + std::to_string(run.input.n50) + "\noutput_reads:\n";
    for (const SubStats& s : outs)
        yaml += "- count: " + std::to_string(s.count) + "\n  bases: " + std::to_string(s.bases) + "\n  n50: " + std::to_string(s.n50) + "\n";
    const std::string yaml_path = out_dir + "/subsample.yaml";
    FILE* y = fopen(yaml_path.c_str(), "wb");
    const bool ok = y && fwrite(yaml.data(), 1, yaml.size(), y) == yaml.size();
    if (!y || fclose(y) != 0 || !ok) throw AcIoError{"cannot write " + yaml_path};
    run.write_ms += ms_since(t0);
    run.kernel_ms = dev.kernel_ms;
    run.copy_ms = dev.copy_ms;
    if (verbose) fprintf(stderr, "\nFinished!\n    You can now assemble each of the subsampled read sets to produce a set of assemblies for input into "
                                 "Autocycler compress.\n\n");
}
