// `autocycler subsample` on the host (subsample.rs): the settings, the genome size, the subset size, the window reader, the seeded
// shuffle, the sample files and subsample.yaml.  The record scan, the statistics and the split into subsets run on the device
// (DeviceSubsample, subsample.cu).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "commands.h"

// parse_genome_size (subsample.rs:83-101): trim, lowercase, Rust's f64 grammar, round half away from zero, a saturating `as u64`, then
// the k/m/g suffixes.  InputError "cannot interpret genome size".
uint64_t parse_genome_size(const std::string& text);
// (0..n).shuffle(&mut StdRng::seed_from_u64(seed)) of rand 0.9 (ChaCha12, IncreasingUniform): order[p] = the read at shuffled position p.
std::vector<uint32_t> subsample_shuffle(uint64_t n, uint64_t seed);
// The first n u32 words of StdRng::seed_from_u64(seed), or of the same generator at another round count (20: ChaCha20).
std::vector<uint32_t> subsample_rng_words(uint64_t seed, uint64_t n, int rounds);

struct SubsampleRun {
    uint64_t genome_size = 0, reads_per_subset = 0, windows = 0, bytes_scanned = 0;
    SubStats input;
    float kernel_ms = 0.f;
    double read_ms = 0, shuffle_ms = 0, write_ms = 0, copy_ms = 0;
};
// The whole command after its settings were checked and out_dir made: pass 1, the statistics, the shuffle, pass 2 and the YAML.
// window: the window size in bytes (it grows for a record longer than it).  InputError for a malformed FASTQ file or too shallow reads,
// std::length_error for 2^32 - 1 reads or a read of 2^32 bases, AcIoError when a file cannot be read or written.
struct AcIoError { std::string msg; };
void subsample_run(DeviceSubsample& dev, const std::string& reads, const std::string& out_dir, uint64_t genome_size, uint64_t count,
                   double min_depth, uint64_t seed, uint64_t window, bool verbose, SubsampleRun& run);
uint64_t subsample_window_size();   // AC_SUBSAMPLE_WINDOW (bytes) or 1 GiB
