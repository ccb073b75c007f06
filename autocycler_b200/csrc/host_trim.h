// `autocycler trim` (trim.rs:36-326) on the host graph, with the overlap alignments on the device (DeviceAlign::overlap_align).
#pragma once
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "host_graph.h"

class DeviceAlign;
struct AlignBatch;

enum TrimMode { TRIM_START_END = 0, TRIM_HAIRPIN_START = 1, TRIM_HAIRPIN_END = 2 };

struct TrimStats {
    float kernel_ms = 0;          // overlap_align kernels, CUDA events (0 under emulation)
    uint32_t rounds = 0;          // overlap_align batches
    uint64_t jobs = 0;            // alignments
    uint64_t cells = 0;           // sum of k^2 over the alignments
    uint32_t max_window = 0;      // largest k
    uint64_t max_path = 0;        // longest path aligned
};

// trim_path_start_end / trim_path_hairpin_start / trim_path_hairpin_end (trim.rs:288-326) for every path of a batch, one device round.
// weights[|unitig|] = unitig length.  trimmed[x] = 0: path x is not trimmed (out[x] is empty).
void trim_paths(DeviceAlign& device, TrimMode mode, const std::vector<std::vector<int32_t>>& paths, const std::vector<uint32_t>& weights,
                double min_identity, uint32_t max_unitigs, std::vector<uint8_t>& trimmed, std::vector<std::vector<int32_t>>& out, TrimStats& stats);

// One cluster of trim_graphs: its graph and sequences (trimmed in place), where its report goes (null: no report) and what its
// alignments were.  stats.kernel_ms is set only when the batch holds this one cluster: a shared launch's time is the batch's.
struct TrimCluster {
    HostGraph* g;
    std::vector<HostSeq>* seqs;
    FILE* log;
    TrimStats stats;
};

// trim_graph for several clusters, phase by phase: every cluster prepares its round-1 pairs, one device round aligns them all, every
// cluster applies its results and prepares round 2, a second device round, then every cluster finishes on its own.  So the device work
// is two overlap_align calls (at most four launches) whatever the number of clusters.
void trim_graphs(DeviceAlign& device, std::vector<TrimCluster>& clusters, double min_identity, uint32_t max_unitigs, double mad, AlignBatch& batch);

// trim.rs:43-51 minus the file I/O: trims the sequences' paths, drops length outliers, cleans up the graph (recalculate_depths,
// remove_zero_depth_unitigs, merge_linear_paths, renumber_unitigs).  `seqs` becomes the kept sequences in their order.  verbose: the
// reference's stderr report.  trim_graphs with one cluster.
void trim_graph(HostGraph& g, std::vector<HostSeq>& seqs, DeviceAlign& device, double min_identity, uint32_t max_unitigs, double mad,
                bool verbose, TrimStats& stats);

// median_isize / mad_isize (misc.rs:399-423), which median_usize / mad_usize equal on lengths
int64_t median_i64(std::vector<int64_t> v);
int64_t mad_i64(const std::vector<int64_t>& v);

// TrimmedClusterMetrics (metrics.rs:209-225) of the sequence lengths, as serde_yaml 0.9 writes it (2_trimmed.yaml)
std::string trimmed_metrics_yaml(const std::vector<HostSeq>& seqs);
