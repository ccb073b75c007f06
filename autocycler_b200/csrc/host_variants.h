// `autocycler variants` on the host: the rule of DESIGN.md §23 around the device's counts, and the texts it writes.  At every position of
// the input it screens the three windows that end in another base, tries polish's candidate edits whose first base there passes the
// screen, and reports those whose k-mers the reads hold at least t times and at a fraction of at least --min_fraction beside the input's
// own k-mers, left-aligned in a VCF.  Not in the reference.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "commands.h"
#include "host_io.h"

// One VCF row: the contig, the left-aligned 1-based POS, the evaluated position p and candidate c, the alleles, and alt, ref and PK.
struct VariantRow {
    uint32_t contig = 0, c = 0, alt = 0, ref = 0, pk = 0;
    uint64_t pos = 0, p = 0;
    std::string ref_allele, alt_allele;
};
struct VariantsResult {
    std::vector<FastaRecord> recs;
    std::vector<VariantRow> rows;
    uint64_t reads = 0, read_windows = 0, read_bases = 0, distinct = 0, valley = 0, min_count = 0, kmers = 0;
    uint64_t positions = 0, screened = 0, candidates = 0, loci = 0, passing = 0;
    uint64_t substitutions = 0, insertions = 0, deletions = 0, paralog = 0, alt_major = 0;
    SpectrumRun spectrum;
    PlRun device;
    VaRun va;
    float kernel_ms = 0.f, scan_ms = 0.f, pack_reads_ms = 0.f;
    double read_ms = 0, copy_ms = 0, host_ms = 0;
};

// The whole rule: the assembly loaded (load_fasta), the reads streamed and packed once and their spectrum counted; t = *min_count, or
// the valley when min_count is null; then the screen, the candidates of edits of up to max_indel bases, and the rows that pass at
// min_fraction.  InputError for an assembly or reads without windows, no valley without min_count, or a malformed file; AcIoError when a
// file cannot be read; std::length_error when the window table or one position's candidate table does not fit.
void variants_run(DeviceSubsample& sub, DeviceSpectrum& spec, DevicePolish& pl, DeviceVariants& dev, const std::string& assembly,
                  const std::string& reads, uint32_t k, const uint32_t* min_count, uint32_t max_indel, double min_fraction, uint64_t window,
                  VariantsResult& out);

// The files under out_dir: variants.vcf and summary.tsv (also the command's stdout).
std::string variants_vcf(const VariantsResult& r);
std::string variants_summary(const VariantsResult& r);
