// `autocycler resolve` (resolve.rs:31-514) on the host graph, with the bridges' all-pairs path distances on the device
// (DeviceAlign::bridge_distances), and `autocycler combine` (combine.rs:25-137), which needs no device.
#pragma once
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "host_graph.h"

class DeviceAlign;
struct AlignBatch;

struct ResolveStats {
    uint32_t anchors = 0;             // anchor unitigs (find_anchor_unitigs, :134-163)
    uint32_t unique_bridges = 0;      // bridges that conflict with no other one after create_bridges
    uint32_t conflicting_bridges = 0;
    uint32_t culled_bridges = 0;      // cull_ambiguity (:285-313)
    uint64_t jobs = 0;                // distance jobs: pairs of distinct trimmed paths of one bridge
    uint64_t cells = 0;               // sum of n * m over the jobs
    uint64_t longest_path = 0;        // longest trimmed path of any bridge (unitigs)
    uint32_t shared_jobs = 0, hbm_jobs = 0;   // jobs whose diagonals sat in shared memory / in HBM scratch
    float kernel_ms = 0;              // bridge_distances kernels, CUDA events (0 under emulation)
};

// Bridge::new (:430-462) for a batch of bridges: groups[g] = the trimmed paths of bridge g (start and end removed), in the reference's
// order, duplicates included.  Identical paths are aligned once, and only pairs of distinct paths go to the device, all groups in one
// round.  totals[g][x] = path x's u32 (wrapping) total of distances to the other paths; best[g] = the path the reference selects (empty
// when every total is u32::MAX).  weights[|unitig|] = unitig length.
void bridge_best_paths(DeviceAlign& device, const std::vector<std::vector<std::vector<int32_t>>>& groups, const std::vector<uint32_t>& weights,
                       std::vector<std::vector<uint32_t>>& totals, std::vector<std::vector<int32_t>>& best, ResolveStats& stats);

// One set of bridges in a batched bridge_best_paths: its groups and weight table, by its own unitig numbers, and its results.  stats
// gains the set's jobs, cells and longest path; the storage-form split and the kernel time only when the batch holds this one set.
struct BridgeSet {
    const std::vector<std::vector<std::vector<int32_t>>>* groups;
    const std::vector<uint32_t>* weights;
    ResolveStats* stats;
    std::vector<std::vector<uint32_t>> totals;
    std::vector<std::vector<int32_t>> best;
};
// bridge_best_paths for several sets at once: their weight tables are concatenated and each set's unitigs rebased onto its part,
// sign * (|u| + base), so all their distance jobs share one bridge_distances call (at most two launches).  A rebased unitig at or above
// 2^31 is a RangeError before any launch.
void bridge_best_paths(DeviceAlign& device, std::vector<BridgeSet>& sets, AlignBatch& batch);

struct ResolveResult { std::string bridged, merged, final_gfa; };    // 3_bridged.gfa, 4_merged.gfa, 5_final.gfa

// One cluster of resolve_texts: the text of its 2_trimmed.gfa, where its report goes (null: no report), its three texts and its counts.
struct ResolveCluster {
    const std::string* text;
    FILE* log;
    ResolveResult out;
    ResolveStats stats;
};
// resolve_text for several clusters, phase by phase: every cluster loads its graph and builds its bridges, one bridge_best_paths call
// aligns all their paths, then every cluster finishes on its own.  With more than one cluster the reports leave the kernel time out.
void resolve_texts(DeviceAlign& device, std::vector<ResolveCluster>& clusters, AlignBatch& batch);

// resolve.rs:41-67 minus the file I/O, on the text of a 2_trimmed.gfa.  verbose: a stderr report of the steps.  resolve_texts with one
// cluster.
void resolve_text(const std::string& trimmed_gfa, DeviceAlign& device, bool verbose, ResolveResult& out, ResolveStats& stats);

// combine.rs:90-137 on the texts of the clusters' final GFAs, in order: consensus_assembly.gfa, .fasta and .yaml (CombineMetrics,
// metrics.rs:229-242, as serde_yaml 0.9 writes it).  verbose: the per-cluster graph summary on stderr.
void combine_texts(const std::vector<std::string>& gfas, const std::vector<std::string>& names, bool verbose, std::string& gfa, std::string& fasta,
                   std::string& yaml);
