// `autocycler helper genome_size` on the host: the window reader, the partition plan and the estimate from the k-mer depth spectrum.
// This departs from the reference on purpose: helper.rs:388-403 runs the Raven assembler over the reads and prints the assembly's total
// length, which this build cannot do.  The number here is a k-mer estimate and will not equal Raven's (DESIGN.md §18).
#pragma once
#include <cstdint>
#include <functional>
#include <string>
#include <vector>

#include "commands.h"

struct GenomeSizeRun {
    uint64_t estimate = 0, reads = 0, bases = 0, windows = 0, distinct = 0, valley = 0, peak = 0, solid = 0;
    double peak_refined = 0;
    uint32_t k = 0;
    SpectrumRun spectrum;
    float kernel_ms = 0.f, scan_ms = 0.f;     // every kernel; the record scan's (the pack, count and histogram are in spectrum)
    double read_ms = 0, copy_ms = 0;
};

// The rule of DESIGN.md §18 on a histogram hist[AC_GS_BINS] of W windows: the valley v, the peak p, the refined peak p* and the estimate
// G = round((W - sum_{c<v} c h[c]) / p*).  Fills every field it names.  InputError when there is no valley (no depth peak) or the error
// k-mers' occurrences exceed W, RangeError when the peak is at the cap or p* is not positive.
void genome_size_rule(const uint64_t* hist, uint64_t windows, GenomeSizeRun& run);

// The valley of hist[AC_GS_BINS]: the smallest c >= 1 whose smoothed sum h[c-1] + h[c] + h[c+1] (h[0] taken as h[1]) is below the next
// one; 0 when there is none.  genome_size_no_peak is the message for that case.
uint64_t genome_size_valley(const uint64_t* hist);
extern const char* const genome_size_no_peak;

// One pass of subsample's windows over a FASTQ file (gzipped or not), each window packed into spec's stream (begun here with k): the
// records, the windows, the time reading and gunzipping the file, and the window uploads' time.  sub.kernel_ms holds the record scan's
// kernels after.  each (when given) runs after each window is packed, with its first record, its records and its first packed word.
struct ReadPass { uint64_t reads = 0, windows = 0; double read_ms = 0, copy_ms = 0; };
ReadPass pack_reads(DeviceSubsample& sub, DeviceSpectrum& spec, const std::string& reads, uint32_t k, uint64_t window,
                    const std::function<void(uint64_t, uint64_t, uint64_t)>& each = nullptr);

// The spectrum of one FASTQ file (gzipped or not): one pass of windows (subsample's scan and messages), each window packed on the
// device, then the partitions counted.  hist gets the AC_GS_BINS bins; genome_size_rule makes the estimate from them.  InputError for a
// malformed file or no k-mer windows, AcIoError when the file cannot be read.
void genome_size_run(DeviceSubsample& sub, DeviceSpectrum& spec, const std::string& reads, uint32_t k, uint64_t window,
                     std::vector<uint64_t>& hist, GenomeSizeRun& run);

// AC_GS_TABLE_SLOTS (the table budget in slots; default a share of free device memory) and AC_GS_PARTITIONS (P; default from the
// budget), read at every call: test switches that reach partitions and reruns on small inputs.
uint64_t genome_size_env(const char* name);
