// `autocycler depth` on the host: the rule of DESIGN.md §19 around the device's counts, the reference's depth filter (helper.rs:889-921)
// and its header parser (helper.rs:923-931), and the texts.  Read-measured depth is an addition that is not in the reference; with
// `--source header` the command is the reference's filter alone.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "commands.h"
#include "host_io.h"

// helper.rs:923-931: the number after the first "depth=", else "depth-", else "coverage=", up to the first '-', '_' or ' ', parsed with
// Rust's f64 grammar.  False when no key is found or the number does not parse.
bool depth_from_header(const std::string& header, double& depth);

// helper.rs:889-921 on loaded records: has[i] says whether record i has a depth.  Returns false, keeping every record and writing
// nothing to report, when neither bound is given or a record has no depth.  Otherwise keep[i] = depth >= threshold, and report gets the
// reference's lines: an empty line, the section's title, "threshold = {:.3}" and "{name}: depth={:.3}, PASS|FAIL" per record.
bool depth_filter(const std::vector<FastaRecord>& recs, const std::vector<double>& depth, const std::vector<char>& has, const double* min_abs,
                  const double* min_rel, std::vector<char>& keep, std::string& report);

// depth_filter on a FASTA text, as the reference applies it to a file: out is what the file holds afterwards.  The text itself when the
// filter does not run or the text holds no bases (is_fasta_empty), the kept records one line per sequence otherwise, and empty when none
// is kept (the reference removes the file).  name stands for the file in load_fasta's messages.
std::string depth_filter_text(const std::string& text, const std::string& name, const double* min_abs, const double* min_rel,
                              std::string& report);

// Rust's `{:.N}` of an f64 (NaN, inf and -inf spelled as Rust does).
std::string rust_fixed(double x, int digits);

// Appends contig r to bytes as the device packs it: its sequence, followed by its first k-1 bases when its header holds
// "circular=true" (any case) and it is at least k long.  Returns its windows of k A/C/G/T bases (shared with qv).
uint64_t pack_contig(const FastaRecord& r, uint32_t k, std::string& bytes);

struct DepthResult {
    std::vector<FastaRecord> recs;
    std::vector<uint64_t> unique;            // per contig: its unique keys
    std::vector<double> depth;               // per contig: the median count (NaN: no depth)
    uint64_t reads = 0, read_windows = 0, read_bases = 0, unique_total = 0;
    DepthRun device;
    float kernel_ms = 0.f, scan_ms = 0.f, pack_reads_ms = 0.f;
    double read_ms = 0, copy_ms = 0;
};
// Reads mode: the assembly (load_fasta) and its headers checked, the table built, the reads streamed through subsample's windows and
// packed (DeviceSpectrum::pack_window), then probed, and each contig's median.  InputError for a header that already carries a depth or a
// malformed file, AcIoError when a file cannot be read, std::length_error when the table does not fit.
void depth_run(DeviceSubsample& sub, DeviceSpectrum& spec, DeviceDepth& dev, const std::string& assembly, const std::string& reads, uint32_t k,
               uint64_t window, DepthResult& out);
