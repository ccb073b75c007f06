// Device pipeline interface (host side).  Replaces the reference's KmerGraph build + unitig walk + link
// creation (compress.rs:42-43 -> kmer_graph.rs:86-134, unitig_graph.rs:176-293, unitig.rs:112-165) with an
// order-free formulation that runs as data-parallel kernels; see DESIGN.md.
#pragma once
#include <cstdint>
#include <functional>
#include <string>
#include <vector>

#include "kmer_key.h"

#define AC_MAX_W 16           // 64-bit words of a k-mer key: k <= 511 (compress.rs:56-58 allows 11..501)
#define AC_MAX_K (32 * AC_MAX_W - 1)
#define AC_MAX_LINKS 5        // successors over the 5-letter alphabet (kmer_graph.rs:142)
#define AC_SEQ_SLACK 32       // spare bytes on both sides of every unitig in the sequence arena

struct PipelineTimings {      // milliseconds, CUDA events on the pipeline's stream (0 under emulation)
    float h2d = 0, pack = 0, sample = 0, insert = 0, insert_kernel = 0, adjacency = 0, boundaries = 0, runs = 0, unitigs = 0, links = 0, seed_sort = 0, emit = 0, simplify = 0, gfa = 0, d2h = 0, total = 0;
};

struct DeviceUnitig {
    uint64_t start;           // global coordinate of the first window of the representative occurrence
    uint32_t len;             // number of k-mers == trimmed length (unitig.rs:157-165)
    uint32_t depth;           // Kmer::depth() of every k-mer in the chain (unitig.rs:148-155)
    uint32_t flip;            // 1: the unitig's forward strand is the reverse complement of the representative occurrence
    int32_t min_d;            // smallest k-mer of both strands (kmer_graph.rs:168-173 order) = the walk's seed
    uint64_t min_w[AC_MAX_W];
    uint32_t head_slot, tail_slot;   // table slots of the representative occurrence's first and last k-mer
};

// One unitig occurrence in rank-independent terms (multi-GPU exchange): where it lies and the smallest occurrence
// of its first and last k-mer.
struct RunRec { uint32_t start, len, head_rep, tail_rep; };     // 16 bytes: coordinates fit 32 bits (inputs are limited to 2^32 - 2 padded bytes)

// The mutable per-unitig state in one 32-byte record (one cache line touch per unitig during repeat expansion).
struct UnitigRec {
    uint64_t seq_off;                          // forward_seq = arena[seq_off, seq_off+len)
    uint32_t len;                              // forward_seq.len()
    uint32_t min_fpos, min_rpos;               // min over forward_positions / reverse_positions (unitig.rs:135-146); all entries shift together
    uint32_t room_before, room_after;          // free arena bytes on both sides (AC_SEQ_SLACK initially)
    uint32_t flags;                            // host scratch
};

// Repeat expansion work list (graph_simplification.rs:43-86): one record per (unitig, side) that can ever shift, listed on the
// device right after the graph is built (links, paths and fixed sets decide it; sequences only enter through spec_len).
struct ExpandCandidate { uint32_t idx; uint16_t side, gn; uint32_t src[6]; };   // 32 B: destination, side (0 inputs / 1 outputs), its sources (UStrand)
struct ExpandDeps { int32_t c[6]; };          // candidates that read unitig u: its own two, and those it exclusively feeds / is fed by

// A unitig strand: (seed index << 1) | reverse.  The seed index is the position the unitig would have had in the
// reference's `unitigs` vector straight after build_unitigs_from_kmer_graph (unitig_graph.rs:179-225).
typedef uint32_t UStrand;

// Everything the host needs, in seed order, living in pinned host memory owned by the pipeline (valid until the
// next build()).  The host edits len / seq_off / min_*pos / arena in place during repeat expansion.
struct PipelineResult {
    uint32_t W = 0;
    uint64_t n_slots_used = 0;                 // distinct canonical k-mers; KmerGraph.kmers.len() == 2x this
    uint64_t capacity = 0;
    uint64_t n_dotted = 0;
    uint64_t h2d_bytes = 0, d2h_bytes = 0;     // bytes copied host->device by upload() and device->host by build()
    uint32_t n_unitigs = 0;
    uint64_t n_runs = 0;
    uint32_t n_seqs = 0;
    UnitigRec* rec = nullptr;                  // [U]
    uint32_t* depth = nullptr;                 // [U]
    uint32_t* order = nullptr;                 // [U] order[n-1] = seed index of unitig number n (renumber_unitigs, unitig_graph.rs:295-315)
    // expand_repeats candidates in the reference's iteration order, with what the host needs to apply them
    uint64_t n_cands = 0;
    ExpandCandidate* cands = nullptr;          // [n_cands]
    uint32_t* spec_len = nullptr;              // [n_cands] length of the common piece of each candidate's sources on the untouched graph
    ExpandDeps* deps = nullptr;                // [U]
    uint8_t* fixed_start = nullptr; uint8_t* fixed_end = nullptr;   // [U] get_fixed_unitig_starts_and_ends (graph_simplification.rs:190-230)
    uint32_t* final_order = nullptr;                                // [U] fused builds: the numbering simplify_structure ends with (:38)
    // The finished file as the device rendered it (fused builds): H, S, L and P lines, pinned
    char* gfa_text = nullptr; uint64_t gfa_bytes = 0;
    // Fused build (DevicePipeline::build(..., fused = true)): simplify_structure and save_gfa ran on the device and only the text and
    // these counts came back; the graph arrays below stay in HBM until fetch_graph() is asked for them.
    bool fused = false, graph_fetched = true;
    uint64_t links_single = 0;                                      // UnitigGraph::link_count().1 (unitig_graph.rs:478-507)
    uint64_t length_before = 0, length_after = 0;                   // total_length() before / after simplify_structure
    char* arena = nullptr; uint64_t arena_used = 0, arena_cap = 0;
    uint32_t* next_off = nullptr;              // [2U+1] CSR over strands: forward_next / reverse_next in the reference's push order
    UStrand* next = nullptr;
    uint32_t* prev_off = nullptr;              // [2U+1] forward_prev / reverse_prev (ascending; only membership matters downstream)
    UStrand* prev = nullptr;
    uint64_t n_links = 0;
    uint64_t* path_off = nullptr;              // [S+1]
    UStrand* path = nullptr;                   // [R] unitig path of every sequence (unitig_graph.rs:447-465)
    uint64_t* run_start = nullptr;             // [R] only when keep_positions: global coordinate / length of every occurrence
    uint32_t* run_len = nullptr;
    PipelineTimings t;
};

// End repair on the device (compress.rs:202-236): every occurrence of one of the k/2-base literals (the fixed halves of the
// 2S repair patterns and their reverse complements) on the forward strands.
struct LiteralHit { uint32_t needle; uint32_t pad; uint64_t gpos; };   // needle index, global coordinate of the matching window

class DevicePipeline {
public:
    DevicePipeline(int device, void* stream);
    ~DevicePipeline();
    // ascii: all padded, end-repaired forward strands concatenated (bytes in "ACGT."); seqs: their layout.
    // seq_lo / seq_hi: copy only the strands of that block of sequences to the device (multi-GPU: every rank uploads its own block and a
    // collective over strand_block() ranges brings the others' over NVLink instead of over every rank's PCIe link).
    void upload(const uint8_t* ascii, uint64_t total, const SeqInfo* seqs, uint32_t n_seqs, uint32_t k, uint32_t seq_lo = 0, uint32_t seq_hi = 0xFFFFFFFFu);
    void* strand_block(uint32_t seq_lo, uint32_t seq_hi, uint64_t* n_bytes);   // device address and size of the strands of sequences [seq_lo, seq_hi) (contiguous)
    // What save_gfa prints around the unitig list of every path (unitig_graph.rs:352-360): "P\t<id>\t" before and
    // "\t*\tLN:i:..\tFN:Z:..\tHD:Z:..\n" behind it, concatenated per sequence (prefix then suffix), with their lengths.  Call before upload().
    void set_path_line_texts(const char* blob, const uint32_t* prefix_len, const uint32_t* suffix_len, uint32_t n_seqs);
    // build() / finish() return once the graph structure is in `out`; the sequence arena and the timings are only valid
    // after complete(), which the caller invokes when it has finished the host work that needs neither.
    void complete(PipelineResult& out);
    // called once per finish(), right before the pinned result buffers are (re)allocated and written (the caller may still be
    // cleaning the previous result out of the CPU caches on other threads)
    std::function<void()> before_results;
    // kernels + D2H of the results (single GPU: all the stages below).  fused: build_kmer_graph, build_unitig_graph,
    // simplify_unitig_graph and the text of save_gfa (compress.rs:42-47) in one device pipeline; only the text comes back.
    void build(PipelineResult& out, bool keep_positions, bool fused = false);
    void fetch_graph(PipelineResult& out, bool keep_positions);   // after a fused build: the graph arrays (simplified, renumbered) into pinned memory
    // Multi-GPU stages (one process per GPU; the collectives between them are done by the caller on device pointers):
    void build_local(uint32_t seq_lo, uint32_t seq_hi, bool multi);     // table over this rank's sequences [seq_lo, seq_hi)
    uint64_t count_entries();                                           // occupied slots of the local table
    void export_entries(void* dst, uint64_t cap_records);               // their 16-byte Slot records, compacted into caller-owned device memory
    void merge_entries(const void* dev_ptr, uint64_t n);                // fold another rank's records into the local table
    void runs_local();                                                  // adjacency + this rank's unitig occurrences
    uint64_t local_runs() const;
    void export_runs(void* dst, uint64_t cap_records);                  // 16-byte RunRec records, ascending coordinate, into caller-owned device memory
    void import_runs(const void* dev_ptr, uint64_t n);                  // rank 0: every rank's records, concatenated in rank order
    // the same from the buffer a padded gather leaves behind: rank r's counts[r] records start at record r * stride
    void import_runs_padded(const void* dev_ptr, uint64_t stride, const uint64_t* counts, uint32_t n_ranks);
    // Several GPUs driven by ONE process (ac_config.n_devices): the exports stay in the exporting pipeline's HBM and the peers' kernels
    // read them in place over NVLink (peer access), so the exchange needs no staging copy and no collective library.
    static void enable_peer_access(const int* devices, int n);          // every device of the set can map every other one's memory
    const void* export_entries_own(uint64_t* n);                        // compacted 16-byte entry records of the local table; valid until the next build
    const void* export_runs_own(uint64_t* n);                           // this rank's 16-byte occurrence records
    void import_runs_from(const void* const* ptrs, const uint64_t* counts, uint32_t n_ranks);   // rank q's records at ptrs[q] (peer memory)
    // unitigs, seeds, links, seed order, host-ready arrays.  split_paths (fused only): the text ends after the L lines; the P lines are
    // printed by the ranks that own the sequences — export_path_tokens() here lays out every occurrence's "(final number - 1) << 1 | strand"
    // for its owner (rank q's tokens at dst + q * stride, counts[q] of them: the occurrence counts the import was given), and every rank
    // turns the tokens of its own occurrences into the P lines of its own sequences (pinned host text) with render_path_lines().
    void finish(PipelineResult& out, bool keep_positions, bool fused = false, bool split_paths = false);
    void export_path_tokens(void* dst, uint64_t stride, const uint64_t* counts, uint32_t n_ranks);
    void render_path_lines(const void* tokens_dev, uint64_t n_tokens, const char** text, uint64_t* bytes);
    // needles: n_needles keys of h bases each (2 words per key, kmer_key.h layout for k = h), pairwise distinct.
    void find_literals(const uint8_t* ascii, uint64_t total, const SeqInfo* seqs, uint32_t n_seqs, uint32_t h,
                       const uint64_t* needle_words, uint32_t n_needles, std::vector<LiteralHit>& hits);
    unsigned long long kernel_launches() const;
    DeviceContext& context();                     // the device and stream the pipeline runs on
    struct Impl;
private:
    Impl* impl;
};
