// `autocycler polish` on the host: the rule of DESIGN.md §22 around the device's counts, and the texts it writes.  Each round finds the
// loci where the reads do not support the consensus, keeps the single-base or short-indel edit that makes every k-mer it touches solid,
// and applies the edits whose spans do not overlap.  Not in the reference.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "commands.h"
#include "host_io.h"

// One row of rounds.tsv: the round's unsupported windows, its loci, and what became of them.
struct PolishRound { uint64_t unsupported = 0, loci = 0, edited = 0, ambiguous = 0, none = 0, edge = 0, deferred = 0; };
struct PolishResult {
    std::vector<FastaRecord> recs;           // the contigs, polished
    std::vector<PolishRound> rounds;
    uint64_t reads = 0, read_windows = 0, read_bases = 0, distinct = 0, valley = 0, min_count = 0;
    uint64_t kmers_before = 0, unsupported_before = 0, kmers_after = 0, unsupported_after = 0, edits = 0;
    std::string edits_tsv, bed;              // edits.tsv without its header, remaining.bed
    SpectrumRun spectrum;
    PlRun device;
    float kernel_ms = 0.f, scan_ms = 0.f, pack_reads_ms = 0.f;
    double read_ms = 0, copy_ms = 0, host_ms = 0;
};

// The whole rule: the assembly loaded (load_fasta), the reads streamed and packed once and their spectrum counted; t = *min_count, or
// the valley when min_count is null; then up to max_rounds rounds of max_indel-base edits, and the polished contigs' windows once more.
// InputError for an assembly or reads without windows, no valley without min_count, or a malformed file; AcIoError when a file cannot
// be read; std::length_error when the tables do not fit.
void polish_run(DeviceSubsample& sub, DeviceSpectrum& spec, DevicePolish& dev, const std::string& assembly, const std::string& reads, uint32_t k,
                const uint32_t* min_count, uint32_t max_indel, uint32_t max_rounds, uint64_t window, PolishResult& out);

// The files under out_dir: polished.fasta, edits.tsv, rounds.tsv and summary.tsv (also the command's stdout); remaining.bed is out.bed.
std::string polish_fasta(const PolishResult& r);
std::string polish_edits(const PolishResult& r);
std::string polish_rounds(const PolishResult& r);
std::string polish_summary(const PolishResult& r, uint32_t k);
