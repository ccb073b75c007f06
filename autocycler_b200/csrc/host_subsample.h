// `autocycler subsample` on the host (subsample.rs): the settings, the genome size, the subset size, the window reader, the seeded
// shuffle, the sample files and subsample.yaml.  The record scan, the statistics and the split into subsets run on the device
// (DeviceSubsample, subsample.cu).
#pragma once
#include <zlib.h>

#include <cstdint>
#include <cstdio>
#include <functional>
#include <string>
#include <vector>

#include "commands.h"

// parse_genome_size (subsample.rs:83-101): trim, lowercase, Rust's f64 grammar, round half away from zero, a saturating `as u64`, then
// the k/m/g suffixes.  InputError "cannot interpret genome size".
uint64_t parse_genome_size(const std::string& text);
// str::parse::<f64> on an already lowercased text: Rust's f64 grammar, nothing else (no hex floats, no partial parses).
bool rust_f64(const std::string& s, double& v);
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

// The FASTQ reader of subsample and genome_size: the file as it is, or gunzipped (every member) when it starts with the gzip magic
// (misc.rs:197-208, 233-245).  AcIoError when it cannot be read, InputError for a broken gzip stream.
struct FastqStream {
    FILE* f = nullptr; gzFile g = nullptr; std::string path;
    explicit FastqStream(const std::string& p);
    FastqStream(const FastqStream&) = delete; FastqStream& operator=(const FastqStream&) = delete;
    ~FastqStream();
    size_t read(uint8_t* dst, size_t n);
};
// One pass over a FASTQ file in windows of at least `window` bytes (it doubles while a window holds no complete record): each window is
// scanned by dev.scan_window (every record checked; the lengths kept when keep_lengths) and each_window(first record, records) runs
// after each scan.  A malformed record is InputError "Error reading FASTQ file: record N: <reason>" (std::length_error for a read of
// 2^32 bases or more).  run.read_ms gets the reading time; with keep_lengths, run.windows and run.bytes_scanned the windows and bytes.
void fastq_windows(DeviceSubsample& dev, const std::string& path, uint64_t& window, bool keep_lengths, SubsampleRun& run,
                   const std::function<void(uint64_t, uint64_t)>& each_window);
