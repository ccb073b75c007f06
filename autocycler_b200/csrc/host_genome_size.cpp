// `autocycler helper genome_size` on the host (see host_genome_size.h and DESIGN.md §18).
#include "host_genome_size.h"

#include <cmath>
#include <cstdlib>

#include "host_io.h"
#include "host_subsample.h"

const char* const genome_size_no_peak = "no k-mer depth peak: the reads are too shallow or too noisy for a k-mer estimate";

uint64_t genome_size_valley(const uint64_t* h) {
    const uint64_t H = AC_GS_BINS;
    // s[c] = h[c-1] + h[c] + h[c+1], with h[0] taken as h[1] (the edge bin repeated: with 0 there, s[1] would sum two bins against
    // s[2]'s three, and any k-mer seen three times would put the valley at 1); the valley is the smallest c >= 1 with s[c] < s[c+1]
    auto s = [&](uint64_t c) { return (c > 1 ? h[c - 1] : h[1]) + h[c] + h[c + 1]; };
    for (uint64_t c = 1; c + 2 < H; ++c)
        if (s(c) < s(c + 1)) return c;
    return 0;
}

void genome_size_rule(const uint64_t* h, uint64_t W, GenomeSizeRun& run) {
    const uint64_t H = AC_GS_BINS;
    run.windows = W;
    run.distinct = 0;
    for (uint64_t c = 1; c < H; ++c) run.distinct += h[c];
    const uint64_t v = genome_size_valley(h);
    if (!v) throw InputError{genome_size_no_peak};
    uint64_t p = v + 1;
    for (uint64_t c = v + 1; c < H - 1; ++c)
        if (h[c] > h[p]) p = c;
    run.valley = v; run.peak = p;
    if (p >= H - 2) throw RangeError{"the k-mer depth peak is at the histogram's cap (" + std::to_string(H - 2) + ")"};
    const int64_t num = (int64_t)h[p - 1] - (int64_t)h[p + 1], den = (int64_t)h[p - 1] - 2 * (int64_t)h[p] + (int64_t)h[p + 1];
    const double ps = den == 0 ? (double)p : (double)p + (double)num / (2.0 * (double)den);
    run.peak_refined = ps;
    uint64_t errors = 0;                              // the occurrences of the k-mers below the valley (exact: every c < v is below the cap)
    for (uint64_t c = 1; c < v; ++c) errors += c * h[c];
    if (errors > W) throw InputError{"the histogram holds more k-mer occurrences below its valley than there are windows"};
    run.solid = W - errors;
    if (!(ps > 0)) throw RangeError{"the refined k-mer depth peak is not positive"};
    const double g = std::round((double)run.solid / ps);
    if (!(g < 18446744073709551616.0)) throw RangeError{"the genome size estimate exceeds 2^64 - 1"};
    run.estimate = (uint64_t)g;
}

uint64_t genome_size_env(const char* name) {
    const char* e = getenv(name);
    return e && *e ? strtoull(e, nullptr, 10) : 0;
}

ReadPass pack_reads(DeviceSubsample& sub, DeviceSpectrum& spec, const std::string& reads, uint32_t k, uint64_t window,
                    const std::function<void(uint64_t, uint64_t, uint64_t)>& each) {
    ReadPass out;
    sub.kernel_ms = 0.f; sub.copy_ms = 0.0;
    spec.begin(k);
    SubsampleRun pass;
    fastq_windows(sub, reads, window, false, pass, [&](uint64_t first, uint64_t records) {
        const uint64_t word0 = spec.packed_words();
        spec.pack_window(sub, records);
        if (each) each(first, records, word0);
        out.reads += records;
        ++out.windows;
    });
    out.read_ms = pass.read_ms;
    out.copy_ms = sub.copy_ms;
    return out;
}

void genome_size_run(DeviceSubsample& sub, DeviceSpectrum& spec, const std::string& reads, uint32_t k, uint64_t window,
                     std::vector<uint64_t>& hist, GenomeSizeRun& run) {
    run = GenomeSizeRun();
    run.k = k;
    const ReadPass pass = pack_reads(sub, spec, reads, k, window);
    run.reads = pass.reads; run.read_ms = pass.read_ms; run.copy_ms = pass.copy_ms;
    spec.totals(&run.windows, &run.bases);
    if (!run.windows) throw InputError{"no k-mer windows: no read holds " + std::to_string(k) + " consecutive A, C, G or T bases"};
    hist.assign(AC_GS_BINS, 0);
    const uint64_t budget = genome_size_env("AC_GS_TABLE_SLOTS");
    spec.count(run.windows, budget ? budget : ac_gs_budget_slots(), genome_size_env("AC_GS_PARTITIONS"), hist.data(), &run.spectrum);
    run.scan_ms = sub.kernel_ms;
    run.kernel_ms = sub.kernel_ms + spec.kernel_ms;
}
