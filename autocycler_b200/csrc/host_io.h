// Stage A of compress on the host (compress.rs:98-133): directory scan, FASTA(.gz) load, padding,
// end repair, and the YAML sidecar (compress.rs:181-189).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "host_graph.h"

struct InputError { std::string msg; };        // the reference's quit_with_error (misc.rs:130-136)
struct RangeError { std::string msg; };        // an input beyond what the device code can index (AC_ERANGE)

struct ContigDetails { std::string name, description; uint64_t length; };
struct AssemblyDetails { std::string filename; std::vector<ContigDetails> contigs; };

struct LoadedInput {
    std::vector<HostSeq> seqs;                 // kept sequences, in id order (start filled by layout())
    std::vector<std::string> padded;           // Sequence.forward_seq: k/2 dots + bases + k/2 dots, after end repair
    uint64_t assembly_count = 0;
    std::vector<AssemblyDetails> details;      // metrics.rs:75-107, includes ignored contigs
};

std::vector<std::string> find_all_assemblies(const std::string& dir);                 // misc.rs:64-95
struct FastaRecord { std::string name, header, seq; };
std::vector<FastaRecord> load_fasta(const std::string& path);                         // misc.rs:144-321
std::string read_fasta_bytes(const std::string& path);                                // the file, gunzipped when it starts with the gzip magic
std::vector<FastaRecord> parse_fasta(const std::string& data, const std::string& path);   // misc.rs:248-321 (load_fasta_allow_empty's parse)
void check_fasta(const std::vector<FastaRecord>& recs, const std::string& path);      // misc.rs:174-194
LoadedInput load_sequences(const std::string& dir, uint32_t k, uint32_t max_contigs, uint32_t threads, bool verbose, DevicePipeline* device);
void sequence_end_repair_device(DevicePipeline& pipe, std::vector<std::string>& padded, uint32_t k);   // compress.rs:202-270, matches found on the GPU
void sequence_end_repair(std::vector<std::string>& padded, uint32_t k, uint32_t threads);   // compress.rs:202-270
std::string metrics_yaml(const LoadedInput& in, uint64_t unitig_count, uint64_t unitig_total_length);  // metrics.rs:65-73,250-254
