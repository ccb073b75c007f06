// Host side of the compress path: everything that operates on unitigs (10^2..10^6 objects, order
// dependent) — link ordering, renumbering, repeat expansion and GFA text.  Input is the device
// pipeline's result; output is byte-identical to the reference's UnitigGraph::save_gfa.
//
// Data layout: structure-of-arrays indexed by the unitig's SEED index (the order in which the
// reference's walk would have created the unitigs, unitig_graph.rs:179-225; it never changes), link
// lists in CSR form per unitig strand, all sequences in one arena with slack on both sides of every
// unitig so that repeat expansion moves bytes without reallocating.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "pipeline.h"

struct HostSeq {              // sequence.rs:19-28 minus the bytes (they live in one concatenated buffer)
    uint16_t id;
    std::string filename, contig_header;
    uint64_t length;          // L
    uint64_t start;           // global coordinate of padded byte 0
    uint16_t cluster = 0;     // Sequence.cluster: 0 on the compress path; carried through from a loaded GFA's CL:i: tag
};

// A unitig strand: (seed index << 1) | reverse (UStrand, pipeline.h).
static inline uint32_t us_index(UStrand s) { return s >> 1; }
static inline bool us_reverse(UStrand s) { return s & 1; }
static inline UStrand us_make(uint32_t idx, bool reverse) { return (idx << 1) | (reverse ? 1u : 0u); }
static inline UStrand us_flip(UStrand s) { return s ^ 1u; }

// "{:.2}" of an f64 depth as the S lines print it (unitig.rs:169); p needs room for 400 bytes.  Returns the length.
uint32_t gfa_depth_text(char* p, double d);

struct HostProfile { double adopt = 0, renumber = 0, candidates = 0, compare = 0, pass1 = 0, expand = 0; int passes = 0; };   // milliseconds (AC_HOST_PROFILE=1 prints them)

class HostGraph {
public:
    uint32_t k = 0;
    uint32_t U = 0;
    // --- per unitig, seed order (unitig.rs:30-45) ---
    // The arrays below are the pipeline's pinned result buffers, adopted and edited in place.
    std::vector<uint32_t> number;             // Unitig.number (1-based position in `order`)
    const uint32_t* depth = nullptr;          // integral on this path: every k-mer of a chain has the same depth
    // Loaded graphs (unitig.rs:62-91) carry what compress never writes: any f64 depth and the segment colour (UnitigType, unitig.rs:385-392).
    // Null for a graph that came from the device; then depth[] is the depth and every unitig is UnitigType::Other.
    const double* depth_f = nullptr;
    const uint8_t* utype = nullptr;           // 0 Other, 1 Anchor, 2 Bridge, 3 Consentig
    double depth_of(uint32_t idx) const { return depth_f ? depth_f[idx] : (double)depth[idx]; }
    uint8_t type_of(uint32_t idx) const { return utype ? utype[idx] : 0; }
    UnitigRec* rec = nullptr;                 // sequence location, length, minimum positions, arena slack (pipeline.h)
    char* arena = nullptr; uint64_t arena_used = 0, arena_cap = 0;
    std::vector<char> arena_overflow;         // only if repeat expansion outgrows the pinned arena
    // --- links, CSR over strands (index 2*idx + reverse): forward_next/reverse_next and forward_prev/reverse_prev ---
    const uint32_t* next_off = nullptr; const uint32_t* prev_off = nullptr;   // [2U+1]
    const UStrand* next = nullptr; const UStrand* prev = nullptr; uint64_t n_links = 0;
    // --- numbering order and paths ---
    std::vector<uint32_t> order;              // order[n-1] = seed index of unitig number n
    const uint64_t* path_off = nullptr;       // [S+1]
    const UStrand* path = nullptr; uint64_t n_path = 0; uint32_t n_seqs = 0;   // get_unitig_path_for_sequence for every sequence (unitig_graph.rs:447-465)
    // optional full position lists (ac_config.keep_positions): CSR per unitig, value = pos << 16 | seq_id_and_strand
    std::vector<uint64_t> fpos_off, rpos_off, fpos, rpos;
    HostProfile prof;

    // unitig_graph.rs:36-48 from the device result (build, simplify_seqs, create_links, trim_overlaps, renumber, check)
    void build(const PipelineResult& r, const std::vector<HostSeq>& seqs, uint32_t k, bool keep_positions);
    void renumber();                          // unitig_graph.rs:295-315
    void check_links() const;                 // unitig_graph.rs:752-793
    void simplify_structure();                // graph_simplification.rs:26-40
    size_t expand_repeats();                  // graph_simplification.rs:43-86
    void prepare_simplify();                  // lists the candidates of expand_repeats ahead of time (links and paths only, no sequence bytes)
    bool adopt_candidates(const PipelineResult& r);   // ... or takes the same lists from a plain build's device result (graph as built only)
    // UnitigGraph::from_gfa_lines (unitig_graph.rs:55-174; host_gfa_load.cpp): replaces the graph by the one in `text`, returns its sequences
    void load_gfa(const char* text, size_t len, std::vector<HostSeq>& seqs);
    void merge_linear_paths(bool use_paths);  // graph_simplification.rs:315-371 (host_merge.cpp); use_paths=false is the reference's `seqs` = [] and drops the paths
    // trim's graph edits (host_trim.cpp).  replace_paths: the sequence paths become `paths` (one per kept sequence, in order) — what
    // remove_sequence_from_graph + create_sequence_and_positions (unitig_graph.rs:151-174, 566-573) do to the positions.
    void replace_paths(const std::vector<std::vector<UStrand>>& paths);
    void recalculate_depths();                // unitig_graph.rs:575-580: depth = forward_positions.len() = path steps through the unitig
    void remove_zero_depth_unitigs();         // unitig_graph.rs:582-586, with delete_dangling_links (:547-564)
    // resolve's graph edits (host_resolve.cpp): the graph becomes these unitigs in this order, with these link lists (index 2 * i + reverse,
    // entries UStrand over the same indices), f64 depths, unitig types and no sequence paths
    void replace_unitigs(const std::vector<uint32_t>& numbers, const std::vector<std::string>& seqs, const std::vector<double>& depths,
                         const std::vector<uint8_t>& types, const std::vector<std::vector<UStrand>>& next_lists, const std::vector<std::vector<UStrand>>& prev_lists);
    // clean's graph edits (host_clean.cpp), on the unitigs in list order; each keeps only the position counts (set_position_counts).
    // Errors: InputError.
    void remove_unitigs(const std::vector<uint32_t>& numbers);   // remove_unitigs_by_number (unitig_graph.rs:588-592)
    void duplicate_unitig(uint32_t num);                         // duplicate_unitig_by_number (:594-668)
    void remove_low_depth_unitigs(double min_depth);             // :670-721
    // what a loaded graph's positions tell merge_linear_paths once clean has edited the graph: counts[i] = forward_positions.len() of
    // unitig i (index order), carried as paths of single steps (the sequences themselves are not kept)
    void set_position_counts(const std::vector<uint32_t>& counts);
    bool is_isolated_and_circular(uint32_t idx) const;           // unitig.rs:275-281: one circularising link and no other
    bool is_isolated_and_linear(uint32_t idx) const;             // :283-292: no links but hairpins
    // unitig_graph.rs:317-360; other_colour: colour_tag(true) (unitig.rs:173-181), Other unitigs get CL:Z:orangered
    void gfa_text(const std::vector<HostSeq>& seqs, std::string& out, bool other_colour = false) const;
    uint64_t total_length() const;
    uint64_t link_count_single() const;       // unitig_graph.rs:478-507 (.1)
    const char* seq_ptr(uint32_t idx) const { return arena + rec[idx].seq_off; }
    const UStrand* next_begin(UStrand s) const { return next + next_off[s]; }
    uint32_t next_size(UStrand s) const { return next_off[s + 1] - next_off[s]; }
    const UStrand* prev_begin(UStrand s) const { return prev + prev_off[s]; }
    uint32_t prev_size(UStrand s) const { return prev_off[s + 1] - prev_off[s]; }
private:
    // storage of the graph once merge_linear_paths has rebuilt it (the pinned pipeline buffers are left behind)
    std::vector<UnitigRec> own_rec; std::vector<uint32_t> own_depth, own_next_off, own_prev_off;
    std::vector<double> own_depth_f; std::vector<uint8_t> own_type;
    std::vector<UStrand> own_next, own_prev, own_path; std::vector<uint64_t> own_path_off;
    std::vector<uint8_t> fixed_start, fixed_end;
    bool fixed_ready = false;
    void compute_fixed();
    // repeat expansion work list: (unitig, side) pairs that satisfy the structural conditions of expand_repeats
    typedef ExpandCandidate Candidate;        // 32 B: destination, side (0 inputs / 1 outputs) and its sources inline (pipeline.h)
    std::vector<Candidate> cands;
    std::vector<int32_t> cand_at;             // [2U] candidate index of (unitig, side), -1 if none
    std::vector<uint64_t> dirty;              // bitmap over cands: must be (re-)evaluated
    std::vector<uint8_t> exhausted;           // per candidate: its sources had nothing in common after its last evaluation
    std::vector<uint32_t> spec_len;           // common-piece lengths computed in parallel at the start of a pass
    std::vector<uint32_t> spec_pass;          // ... and the pass they were computed for
    uint32_t pass_id = 0;                     // expand_repeats calls so far; rec[].flags holds the pass a unitig last changed in
    bool cands_ready = false, first_pass = true;
    void compute_candidates();
    bool spec_from_device = false;
    uint32_t common_length(const Candidate& cand) const;
    // The sources of a candidate: its inline copy (at most 6; a graph built from k-mers has at most 5 neighbours per side), or, for
    // a loaded graph with more, the link list they were copied from (links never change during simplify_structure).
    const UStrand* sources(const Candidate& cand) const {
        return cand.gn <= 6 ? cand.src : (cand.side == 0 ? prev_begin(us_make(cand.idx, false)) : next_begin(us_make(cand.idx, false)));
    }
    typedef ExpandDeps Deps;                  // candidates that read unitig u (pipeline.h)
    std::vector<Deps> deps;
    void compute_dependents();
    static constexpr size_t POSTPONED = (size_t)-1;   // apply_candidate: the shared arena was full, nothing was changed
    size_t apply_candidate(size_t ci, bool shared, std::string& common);
    std::vector<uint32_t> level_start, by_level; uint32_t n_levels = 0;   // candidates grouped by conflict level (compute_levels)
    size_t last_evaluations = 0;
    void compute_levels();
    size_t pass_parallel(bool all_due);
    void reserve_arena(uint64_t extra);
    bool relocate(uint32_t idx, uint32_t before, uint32_t after, bool shared);
};
