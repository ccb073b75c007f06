// `autocycler cluster` (cluster.rs:30-912) after the distances: the tree from the device's UPGMA merge list, normalisation and Newick,
// automatic clustering refined by score or manual clustering, QC, reordering, and the text of every output file.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "host_graph.h"

class DeviceCluster;

struct ClusterStats {
    float distance_ms = 0, upgma_ms = 0;     // distance and UPGMA kernels, CUDA events (0 under emulation)
    double cluster_gfa_ms = 0;                // host time of the per-cluster 1_untrimmed.gfa files (save_cluster_gfa, :794-806)
    uint32_t n_seqs = 0, pass_clusters = 0, fail_clusters = 0;
};

struct ClusterResult {
    std::string phylip, newick, tsv, yaml;    // pairwise_distances.phylip, clustering.newick, clustering.tsv, clustering.yaml
    std::vector<uint16_t> seq_cluster;        // per sequence (the handle's order): its cluster number (1-based, after reordering)
    std::vector<uint8_t> cluster_pass;        // per cluster c - 1
    std::vector<std::string> cluster_gfa, cluster_yaml;   // per cluster c - 1: 1_untrimmed.gfa and 1_untrimmed.yaml
};

// The whole of cluster.rs:42-59 on a graph loaded from `gfa` (the text of input_assemblies.gfa; `g` and `seqs` are its load_gfa result).
// min_assemblies < 0: set automatically (set_min_assemblies, :645-661).  manual: parsed node numbers, sorted (empty = automatic).
// Errors (InputError): the reference's messages, and a clean error where the reference would panic on NaN distances (two sequences
// whose paths have no length).  verbose: the reference's stderr report, without colours.
// `gfa` must describe the same graph as `g` (the reference re-loads it per cluster).  seqs[].cluster is set to the clusters.
// out_dir: the clustering directory the verbose report names.
void cluster_graph(const std::string& gfa, const HostGraph& g, std::vector<HostSeq>& seqs, DeviceCluster& device, double cutoff, int64_t min_assemblies,
                   const std::vector<uint16_t>& manual, uint32_t max_contigs, const std::string& out_dir, bool verbose, ClusterResult& out, ClusterStats& stats);

// Sequence::consensus_weight (sequence.rs:104-109): the autocycler_consensus_weight= value of the header, 1 when absent or unparsable
uint64_t sequence_consensus_weight(const HostSeq& s);

// parse_manual_clusters (:664-671): "1, 2,3" -> sorted node numbers
std::vector<uint16_t> parse_manual_clusters(const std::string& text);

// save_distance_matrix (:160-174): the count, then per sequence its Display form (sequence.rs:112-135) and the distances with 8 decimals
std::string distance_matrix_text(const std::vector<HostSeq>& seqs, const double* d);

// Number formats of the output files: Rust's `{}` for f64 (shortest round trip, never an exponent), serde_yaml 0.9's f64 (ryu's
// layout), and format_float (misc.rs:363-370: `{:.6}` without trailing zeros)
std::string rust_display_f64(double v);
std::string yaml_f64(double v);
std::string format_float(double v);
