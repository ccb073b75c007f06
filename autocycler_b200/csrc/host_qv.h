// `autocycler qv` on the host: the rule of DESIGN.md §20 around the device's counts, and the texts it writes.  Each assembly's k-mer QV
// (the share of its windows whose key the reads hold fewer than t times) and completeness (the share of the reads' solid keys it holds),
// per assembly and per contig, the unsupported stretches as BED and Merqury's copy-number spectrum.  Not in the reference.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "commands.h"
#include "host_io.h"

struct QvContig { std::string name; uint64_t length = 0, kmers = 0, unsupported = 0; };
struct QvAssembly {
    std::string path;                        // as given, or as find_all_assemblies returned it
    std::vector<QvContig> contigs;
    uint64_t kmers = 0, unsupported = 0, solid_found = 0;
    std::string bed, spectrum;               // unsupported/<n>.bed and spectra_cn/<n>.tsv
};
struct QvResult {
    std::vector<QvAssembly> assemblies;
    std::vector<uint64_t> hist;              // the reads' AC_GS_BINS bins, as genome_size counts them
    uint64_t reads = 0, read_windows = 0, read_bases = 0, distinct = 0, valley = 0, min_count = 0, solid = 0;
    SpectrumRun spectrum;
    QvRun device;
    float kernel_ms = 0.f, scan_ms = 0.f, pack_reads_ms = 0.f;
    double read_ms = 0, copy_ms = 0;
};

// The assemblies the arguments name, in order: a directory expands to find_all_assemblies' files, a file stays as given.  InputError
// for a path that does not exist or a directory without assemblies.
std::vector<std::string> qv_inputs(const std::vector<std::string>& args);

// The whole rule: the assemblies loaded (load_fasta), their keys claimed in the combined table, the reads streamed and packed once,
// probed, and their spectrum counted; t = *min_count, or the valley when min_count is null; then each assembly's passes and texts.
// InputError for an assembly without windows, reads without windows, no valley without min_count, or a malformed file; AcIoError when a
// file cannot be read; std::length_error when the tables do not fit.
void qv_run(DeviceSubsample& sub, DeviceSpectrum& spec, DeviceQv& dev, const std::vector<std::string>& assemblies, const std::string& reads,
            uint32_t k, const uint32_t* min_count, uint64_t window, QvResult& out);

// One contig's BED lines (appended to bed) from its masks, one u32 per packed word of its L bases and junction bases: each unsupported
// window ending at e covers [e-k+1, e], split at the end of a circular contig's sequence; touching and overlapping intervals merged.
void contig_bed(const std::string& name, uint64_t L, const uint32_t* mask, uint64_t words, uint32_t k, std::string& bed);
// -10 log10(p), p = -expm1(log1p(-E / K) / k), as `%.2f`; "inf" for E = 0 and "" for K = 0.
std::string qv_text(uint64_t unsupported, uint64_t kmers, uint32_t k);
// The files under out_dir: qv.tsv, contig_qv.tsv and kmer_histogram.tsv (the BED and spectrum texts are in each QvAssembly).
std::string qv_table(const QvResult& r, uint32_t k);
std::string qv_contig_table(const QvResult& r, uint32_t k);
std::string qv_histogram(const QvResult& r);
