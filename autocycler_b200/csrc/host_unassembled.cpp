// `autocycler unassembled` on the host (see host_unassembled.h and DESIGN.md §21).
#include "host_unassembled.h"

#include <chrono>
#include <cstdio>
#include <cstring>
#include <stdexcept>

#include "host_depth.h"
#include "host_genome_size.h"
#include "host_subsample.h"

namespace {
double ms_since(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

std::string fixed(const char* format, double x) {
    char buf[64];
    snprintf(buf, sizeof buf, format, x);
    return buf;
}

// The start of each unassembled.tsv row from gathered records `@head\nseq\n+\nqual\n`: the header up to its first space or tab, and the
// sequence length.
void table_rows(const uint8_t* p, uint64_t n, std::vector<std::string>& rows) {
    for (uint64_t i = 0; i < n;) {
        const uint8_t* head = p + i + 1;
        const uint8_t* head_end = (const uint8_t*)memchr(head, '\n', n - i - 1);
        const uint8_t* seq_end = (const uint8_t*)memchr(head_end + 1, '\n', p + n - head_end - 1);
        const uint64_t len = (uint64_t)(seq_end - head_end - 1);
        const uint8_t* name_end = head;
        while (name_end < head_end && *name_end != ' ' && *name_end != '\t') ++name_end;
        rows.push_back(std::string((const char*)head, (size_t)(name_end - head)) + "\t" + std::to_string(len) + "\t");
        i = (uint64_t)(seq_end - p) + 3 + len + 1;          // "\n+\n", the quality, "\n"
    }
}
}  // namespace

void unassembled_run(DeviceSubsample& sub, DeviceSpectrum& spec, DeviceUnassembled& dev, const std::vector<std::string>& paths,
                     const std::string& reads, uint32_t k, const uint32_t* min_count, uint64_t min_solid, double min_fraction, uint64_t window,
                     const std::string& out_dir, UnassembledResult& out) {
    out = UnassembledResult();
    out.paths = paths;
    // every input's contigs back to back: together they are the assembly
    std::string bytes;
    std::vector<uint64_t> len;
    uint64_t windows = 0;
    for (const std::string& path : paths)
        for (const FastaRecord& r : load_fasta(path)) {
            const size_t start = bytes.size();
            windows += pack_contig(r, k, bytes);
            len.push_back(bytes.size() - start);
        }
    if (len.size() >= 0xFFFFFFFFull) throw RangeError{"unassembled: 2^32 - 1 contigs or more"};
    if (!windows) {
        std::string names;
        for (const std::string& p : paths) names += (names.empty() ? "" : ", ") + p;
        throw InputError{"no k-mer windows: no contig of " + names + " holds " + std::to_string(k) + " consecutive A, C, G or T bases"};
    }
    out.contigs = len.size();
    const uint64_t budget_env = genome_size_env("AC_UNASSEMBLED_TABLE_SLOTS");
    const uint64_t budget_slots = budget_env ? budget_env : ac_gs_budget_slots();
    dev.build((const uint8_t*)bytes.data(), len.data(), (uint32_t)len.size(), windows, k, budget_slots, &out.device);
    const ReadPass pass = pack_reads(sub, spec, reads, k, window, [&](uint64_t first, uint64_t records, uint64_t word0) {
        dev.index_window(spec, sub, first, records, word0, &out.device);
    });
    out.reads = pass.reads; out.windows = pass.windows; out.read_ms = pass.read_ms; out.copy_ms = pass.copy_ms;
    spec.totals(&out.read_windows, &out.read_bases);
    if (!out.read_windows) throw InputError{"no k-mer windows: no read holds " + std::to_string(k) + " consecutive A, C, G or T bases"};
    dev.check_budget(out.reads, spec.packed_words(), budget_slots, &out.device);
    out.hist.assign(AC_GS_BINS, 0);
    const uint64_t budget = genome_size_env("AC_GS_TABLE_SLOTS");          // read after the set and the counters exist: half of what is left
    spec.count(out.read_windows, budget ? budget : ac_gs_budget_slots(), genome_size_env("AC_GS_PARTITIONS"), out.hist.data(), &out.spectrum);
    const uint64_t* h = out.hist.data();
    for (uint64_t c = 1; c < AC_GS_BINS; ++c) out.distinct += h[c];
    out.valley = genome_size_valley(h);
    if (!min_count && !out.valley)
        throw InputError{std::string(genome_size_no_peak) + "; --min_count sets the solid threshold without it"};
    const uint64_t t = min_count ? *min_count : out.valley;
    out.min_count = t;
    try {
        GenomeSizeRun gs;
        genome_size_rule(h, out.read_windows, gs);
        out.peak = gs.peak_refined; out.has_peak = true;
    } catch (const InputError&) {
    } catch (const RangeError&) {}
    // the attribution sweep, then the rule per read
    std::vector<uint32_t> counts(2 * out.reads), lengths(out.reads);
    out.absent.assign(AC_GS_BINS, 0);
    dev.attribute(spec, out.reads, (uint32_t)t, counts.data(), lengths.data(), out.absent.data(), &out.device);
    out.fraction_reads.assign(101, 0); out.fraction_bases.assign(101, 0);
    std::vector<uint32_t> order;
    order.reserve(out.reads);
    std::vector<uint32_t> solid_of, absent_of;                   // the selected reads' s and a, in input order
    for (uint64_t i = 0; i < out.reads; ++i) {
        const uint64_t s = counts[2 * i], a = counts[2 * i + 1];
        if (s < min_solid) continue;
        ++out.scored;
        const uint64_t b = 100 * a / s;
        ++out.fraction_reads[b]; out.fraction_bases[b] += lengths[i];
        if ((double)a >= min_fraction * (double)s) {
            order.push_back((uint32_t)i);
            solid_of.push_back((uint32_t)s); absent_of.push_back((uint32_t)a);
            ++out.selected; out.selected_bases += lengths[i];
        }
    }
    for (uint64_t c = 1; c < AC_GS_BINS; ++c) out.absent_kmers += out.absent[c];
    if (out.absent_kmers) {                                      // the middle bin value, or the mean of the two middle ones
        const uint64_t lo = (out.absent_kmers - 1) / 2, hi = out.absent_kmers / 2;
        uint64_t seen = 0, v_lo = 0, v_hi = 0;
        for (uint64_t c = 1; c < AC_GS_BINS; ++c) {
            if (seen <= lo && lo < seen + out.absent[c]) v_lo = c;
            if (seen <= hi && hi < seen + out.absent[c]) { v_hi = c; break; }
            seen += out.absent[c];
        }
        out.absent_median = ((double)v_lo + (double)v_hi) / 2.0; out.has_median = true;
    }
    // unassembled.fastq: subsample's gather with the selected reads first in the order, the window still on the device when there was
    // one, else the file read again
    const std::string fastq = out_dir + "/unassembled.fastq";
    FILE* f = fopen(fastq.c_str(), "wb");
    if (!f) throw AcIoError{"cannot write " + fastq};
    struct Closer { FILE*& f; ~Closer() { if (f) fclose(f); } } closer{f};
    out.table = "read\tlength\tsolid_kmers\tabsent_kmers\n";
    std::vector<std::string> rows;
    if (out.selected) {
        std::vector<uint8_t> chosen(out.reads, 0);
        for (uint32_t i : order) chosen[i] = 1;
        for (uint64_t i = 0; i < out.reads; ++i) if (!chosen[i]) order.push_back((uint32_t)i);
        const float before = sub.kernel_ms;
        sub.set_order(order.data(), out.reads);
        auto write_window = [&](uint64_t first, uint64_t) {
            sub.h_out.ensure(std::max<uint64_t>(sub.h_win.cap, 1) + 1);
            const uint64_t n = sub.gather(first, out.reads, 0, out.selected, sub.h_out.as<uint8_t>());
            const auto t0 = std::chrono::steady_clock::now();
            table_rows(sub.h_out.as<uint8_t>(), n, rows);
            if (n && fwrite(sub.h_out.p, 1, n, f) != n) throw AcIoError{"cannot write " + fastq};
            out.write_ms += ms_since(t0);
        };
        if (out.windows == 1) write_window(0, out.reads);
        else {
            SubsampleRun again;
            fastq_windows(sub, reads, window, false, again, write_window);
            out.read_ms += again.read_ms;
        }
        out.gather_ms = sub.kernel_ms - before;
    }
    if (rows.size() != out.selected) throw std::logic_error("unassembled: the gathered records are not the selected reads");
    for (uint64_t j = 0; j < out.selected; ++j)
        out.table += rows[j] + std::to_string(solid_of[j]) + "\t" + std::to_string(absent_of[j]) + "\n";
    const auto t0 = std::chrono::steady_clock::now();
    const bool good = fclose(f) == 0;
    f = nullptr;
    if (!good) throw AcIoError{"cannot write " + fastq};
    out.write_ms += ms_since(t0);
    out.scan_ms = sub.kernel_ms - out.gather_ms;
    out.pack_reads_ms = spec.packed_ms();
    out.kernel_ms = sub.kernel_ms + spec.kernel_ms + out.device.pack_ms + out.device.claim_ms + out.device.index_ms + out.device.sweep.count_ms +
                    out.device.attribute_ms;
}

std::string unassembled_median_text(const UnassembledResult& r) { return r.has_median ? fixed("%.1f", r.absent_median) : ""; }
std::string unassembled_peak_text(const UnassembledResult& r) { return r.has_peak ? fixed("%.2f", r.peak) : ""; }
std::string unassembled_ratio_text(const UnassembledResult& r) {
    return r.has_median && r.has_peak ? fixed("%.2f", r.absent_median / r.peak) : "";
}

std::string unassembled_summary(const UnassembledResult& r) {
    return "reads\tread_windows\tmin_count\tscored_reads\tselected_reads\tselected_bases\tabsent_kmers\tabsent_median\tpeak\tabsent_copy_ratio\n" +
           std::to_string(r.reads) + "\t" + std::to_string(r.read_windows) + "\t" + std::to_string(r.min_count) + "\t" + std::to_string(r.scored) +
           "\t" + std::to_string(r.selected) + "\t" + std::to_string(r.selected_bases) + "\t" + std::to_string(r.absent_kmers) + "\t" +
           unassembled_median_text(r) + "\t" + unassembled_peak_text(r) + "\t" + unassembled_ratio_text(r) + "\n";
}

std::string unassembled_fractions(const UnassembledResult& r) {
    std::string t = "percent\treads\tbases\n";
    for (uint32_t b = 0; b <= 100; ++b)
        t += std::to_string(b) + "\t" + std::to_string(r.fraction_reads[b]) + "\t" + std::to_string(r.fraction_bases[b]) + "\n";
    return t;
}

namespace {
std::string bins_text(const std::vector<uint64_t>& h) {     // kmer_histogram.tsv's layout: `count<TAB>k-mers`, the non-zero bins
    std::string t;
    for (uint64_t c = 1; c < AC_GS_BINS; ++c)
        if (h[c]) t += std::to_string(c) + "\t" + std::to_string(h[c]) + "\n";
    return t;
}
}  // namespace

std::string unassembled_absent(const UnassembledResult& r) { return bins_text(r.absent); }
std::string unassembled_kmer_histogram(const UnassembledResult& r) { return bins_text(r.hist); }
