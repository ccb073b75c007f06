// `autocycler unassembled` on the host: the rule of DESIGN.md §21 around the device's counts, and the texts it writes.  For each read,
// its solid windows (the reads hold their key t times or more) and how many of them the assembly lacks; the reads where that share is
// high, written as FASTQ; and the solid keys the assembly lacks, binned by read count and set against the genome's k-mer peak.  Not in
// the reference.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "commands.h"
#include "host_io.h"

struct UnassembledResult {
    std::vector<std::string> paths;          // the assembly files, as qv_inputs expanded them
    uint64_t contigs = 0, reads = 0, windows = 0, read_windows = 0, read_bases = 0, distinct = 0, valley = 0, min_count = 0;
    uint64_t scored = 0, selected = 0, selected_bases = 0, absent_kmers = 0;
    bool has_median = false, has_peak = false;
    double absent_median = 0, peak = 0;
    std::vector<uint64_t> hist, absent;      // the reads' AC_GS_BINS bins, and the absent keys' bins
    std::vector<uint64_t> fraction_reads, fraction_bases;       // 101 rows
    std::string table;                       // unassembled.tsv
    SpectrumRun spectrum;
    UaRun device;
    float kernel_ms = 0.f, scan_ms = 0.f, pack_reads_ms = 0.f, gather_ms = 0.f;
    double read_ms = 0, copy_ms = 0, write_ms = 0;
};

// The whole rule: the assemblies loaded (load_fasta) and their keys claimed in one set, the reads streamed and packed once with each
// word's read index, their spectrum counted; t = *min_count, or the valley when min_count is null; then the attribution sweep, the
// selection and out_dir/unassembled.fastq (out_dir must exist).  InputError for an assembly without windows, reads without windows, no
// valley without min_count, or a malformed file; AcIoError when a file cannot be read or written; std::length_error when the tables do
// not fit.
void unassembled_run(DeviceSubsample& sub, DeviceSpectrum& spec, DeviceUnassembled& dev, const std::vector<std::string>& assemblies,
                     const std::string& reads, uint32_t k, const uint32_t* min_count, uint64_t min_solid, double min_fraction, uint64_t window,
                     const std::string& out_dir, UnassembledResult& out);

// The other files under out_dir: summary.tsv (also the command's stdout), fraction_histogram.tsv, absent_histogram.tsv and
// kmer_histogram.tsv (unassembled.tsv is out.table).
std::string unassembled_summary(const UnassembledResult& r);
std::string unassembled_fractions(const UnassembledResult& r);
std::string unassembled_absent(const UnassembledResult& r);
std::string unassembled_kmer_histogram(const UnassembledResult& r);
// The summary's absent_median, peak and absent_copy_ratio fields: `%.1f`, `%.2f` and `%.2f`, empty when not defined.
std::string unassembled_median_text(const UnassembledResult& r);
std::string unassembled_peak_text(const UnassembledResult& r);
std::string unassembled_ratio_text(const UnassembledResult& r);
