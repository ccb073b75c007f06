// ORACLE — TEST INFRASTRUCTURE ONLY.
//
// CPU restatement (C++17) of the reference's `autocycler compress` hot path, written from reading
// rrwick/Autocycler v0.6.1 (Rust).  Each function cites the reference file:line it follows.
// Nothing in the product (autocycler_b200/, include/) may include, link or execute this; only
// tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it,
// and only as the checker / timed CPU baseline.
//
// Parity pinning: the reference cannot be compiled here (no Rust toolchain, crates not vendored), and
// it ships no golden compress output.  The oracle is pinned by every KAT the reference's own tests hold
// for this path (tests/test_oracle_kats.py lists them with file:line) and by the reference's two
// end-to-end invariants (src/tests.rs:75-167: GFA save->load->save identity and exact reconstruction).
// Byte-level GFA parity with the Rust binary itself is therefore "parity unpinned" beyond those.
#pragma once
#include <cstdint>
#include <deque>
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>

namespace orc {

[[noreturn]] void quit_with_error(const std::string& text);   // misc.rs:130-141 (throws OracleError)

struct OracleError { std::string msg; };

namespace strand { constexpr bool FORWARD = true; constexpr bool REVERSE = false; }  // misc.rs:26-30

// position.rs:18-52
struct Position {
    uint32_t pos;
    uint16_t seq_id_and_strand;
    static constexpr uint16_t STRAND_BIT_MASK = 0x8000;
    Position(uint16_t seq_id, bool strand, size_t p)
        : pos((uint32_t)p), seq_id_and_strand(strand ? (uint16_t)(seq_id | STRAND_BIT_MASK) : seq_id) {}
    uint16_t seq_id() const { return seq_id_and_strand & (uint16_t)~STRAND_BIT_MASK; }
    bool strand() const { return (seq_id_and_strand & STRAND_BIT_MASK) != 0; }
    std::string to_string() const;
};

// sequence.rs:19-59
struct Sequence {
    uint16_t id = 0;
    std::string forward_seq, reverse_seq;
    std::string filename, contig_header;
    size_t length = 0;
    uint16_t cluster = 0;
    static Sequence new_with_seq(size_t id, std::string seq, std::string filename, std::string contig_header,
                                 size_t length, uint32_t half_k);
    static Sequence new_without_seq(uint16_t id, std::string filename, std::string contig_header, size_t length,
                                    uint16_t cluster);
    std::string contig_name() const;
    std::string contig_description() const;
    bool is_ignored() const;
    bool is_trusted() const;
    std::string display() const;
    size_t cluster_weight() const;      // sequence.rs:96-101
    size_t consensus_weight() const;    // sequence.rs:103-108
};

std::string reverse_complement(const std::string& s);                       // misc.rs:324-342
std::vector<std::string> find_all_assemblies(const std::string& dir);       // misc.rs:64-95
std::vector<std::tuple<std::string, std::string, std::string>> load_fasta(const std::string& filename);  // misc.rs:144-321

// metrics.rs:65-107
struct InputContigDetails { std::string name, description; uint64_t length; };
struct InputAssemblyDetails { std::string filename; std::vector<InputContigDetails> contigs; };
struct InputAssemblyMetrics {
    uint32_t input_assemblies_count = 0, input_assemblies_total_contigs = 0;
    uint64_t input_assemblies_total_length = 0;
    uint32_t compressed_unitig_count = 0;
    uint64_t compressed_unitig_total_length = 0;
    std::vector<InputAssemblyDetails> input_assembly_details;
    std::string to_yaml() const;                                            // metrics.rs:250-254 (serde_yaml 0.9)
};

// compress.rs:98-133, 202-270
std::pair<std::vector<Sequence>, size_t> load_sequences(const std::string& assemblies_dir, uint32_t k_size,
                                                        InputAssemblyMetrics& metrics, uint32_t max_contigs,
                                                        int threads, bool verbose);
void sequence_end_repair(std::vector<Sequence>& sequences, uint32_t k_size, int threads);
std::string find_best_match(const std::vector<std::string>& matches);

// kmer_graph.rs:26-61
struct Kmer {
    const char* pointer;
    size_t length;
    std::vector<Position> positions;
    bool seen = false;   // stands in for the reference's `seen: HashSet<&[u8]>` (unitig_graph.rs:177)
    std::string seq() const { return std::string(pointer, length); }
    size_t depth() const { return positions.size(); }
    bool first_position() const { for (auto& p : positions) if (p.pos == 0) return true; return false; }
    std::string display() const;
    size_t cluster_weight() const;      // sequence.rs:96-101
    size_t consensus_weight() const;    // sequence.rs:103-108
};

// kmer_graph.rs:73-181
class KmerGraph {
public:
    uint32_t k_size;
    explicit KmerGraph(uint32_t k) : k_size(k) {}
    void add_sequences(const std::vector<Sequence>& seqs, size_t assembly_count);
    void add_sequence(const Sequence& seq, size_t assembly_count);
    std::vector<Kmer*> next_kmers(const char* kmer) ;
    std::vector<Kmer*> prev_kmers(const char* kmer) ;
    std::vector<Kmer*> iterate_kmers();
    Kmer* reverse(const Kmer* kmer);
    Kmer* get(const char* key);
    size_t len() const { return kmers.size(); }
private:
    // open-addressing map keyed on the k bytes behind `pointer` (stands in for FxHashMap<&[u8], Kmer>)
    std::deque<Kmer> kmers;
    std::vector<uint32_t> table;   // index+1 into kmers, 0 = empty
    size_t mask = 0;
    uint64_t hash(const char* p) const;
    Kmer* entry(const char* key, size_t assembly_count, bool* created);
    void grow();
};

struct Unitig;
struct UnitigStrand { Unitig* unitig; bool strand; uint32_t number() const; };

enum class UnitigType { Anchor, Bridge, Consentig, Other };   // unitig.rs:385-392 (default Other)

// unitig.rs:30-248
struct Unitig {
    uint32_t number = 0;
    UnitigType unitig_type = UnitigType::Other;
    std::deque<Kmer*> forward_kmers, reverse_kmers;
    std::string forward_seq, reverse_seq;
    double depth = 0.0;
    std::vector<Position> forward_positions, reverse_positions;
    std::vector<UnitigStrand> forward_next, forward_prev, reverse_next, reverse_prev;
    static Unitig from_kmers(uint32_t number, Kmer* f, Kmer* r);
    static Unitig from_segment_line(const std::string& line);
    void add_kmer_to_end(Kmer* f, Kmer* r);
    void add_kmer_to_start(Kmer* f, Kmer* r);
    void simplify_seqs();
    void trim_overlaps(size_t k_size);
    std::string gfa_segment_line() const;
    uint32_t length() const { return (uint32_t)forward_seq.size(); }
    const std::string& get_seq(bool strand) const { return strand ? forward_seq : reverse_seq; }
    void remove_seq_from_start(size_t amount);
    void remove_seq_from_end(size_t amount);
    void add_seq_to_start(const std::string& seq);
    void add_seq_to_end(const std::string& seq);
};

// unitig_graph.rs:28-516, 723-793
class UnitigGraph {
public:
    std::vector<std::unique_ptr<Unitig>> unitigs;
    uint32_t k_size = 0;
    std::unordered_map<uint32_t, Unitig*> unitig_index;

    static UnitigGraph from_kmer_graph(KmerGraph& kg);
    static std::pair<UnitigGraph, std::vector<Sequence>> from_gfa_lines(const std::vector<std::string>& lines);
    void build_unitig_index();
    void renumber_unitigs();
    void check_links() const;
    std::string gfa_text(const std::vector<Sequence>& sequences) const;   // save_gfa, unitig_graph.rs:317-331
    std::vector<std::pair<uint32_t, bool>> get_unitig_path_for_sequence(const Sequence& seq) const;
    std::string reconstruct_original_sequence(const Sequence& seq) const;
    uint64_t total_length() const;
    std::pair<size_t, size_t> link_count() const;
    bool link_exists(uint32_t a, bool as, uint32_t b, bool bs) const;
    bool link_exists_prev(uint32_t a, bool as, uint32_t b, bool bs) const;
    void delete_dangling_links();                                           // unitig_graph.rs:547-564
    uint32_t max_unitig_number() const;                                     // unitig_graph.rs:901-903
    std::vector<std::vector<uint32_t>> connected_components() const;        // unitig_graph.rs:905-947
    bool component_is_circular_loop(const std::vector<uint32_t>& component) const;   // unitig_graph.rs:949-967
    // Unitigs dropped from `unitigs` stay alive here until the graph dies: the reference holds them through Rc, and
    // links to them are still walked (by number) until delete_dangling_links has run.
    std::vector<std::unique_ptr<Unitig>> retired;

    // stages of from_kmer_graph, public so tests can inspect the pre-renumber ("seed order") state
    void build_unitigs_from_kmer_graph(KmerGraph& kg);
    void simplify_seqs();
    void create_links();
    void trim_overlaps();
private:
    UnitigStrand find_starting_unitig(uint16_t seq_id) const;
    // (seq_id, strand, pos) of every entry of a long position list, built the first time one walk along a sequence looks the list up
    typedef std::unordered_map<const std::vector<Position>*, std::unordered_set<uint64_t>> PositionIndex;
    bool get_next_unitig(uint16_t seq_id, bool seq_strand, const Unitig* u, bool strand, uint32_t pos,
                         UnitigStrand* next, uint32_t* next_pos, PositionIndex* index = nullptr) const;
};

// graph_simplification.rs:26-312
void simplify_structure(UnitigGraph& graph, const std::vector<Sequence>& seqs);
size_t expand_repeats(UnitigGraph& graph, const std::vector<Sequence>& seqs);
std::vector<UnitigStrand> get_exclusive_inputs(const Unitig* u);
std::vector<UnitigStrand> get_exclusive_outputs(const Unitig* u);
std::string get_common_start_seq(const std::vector<UnitigStrand>& unitigs);
std::string get_common_end_seq(const std::vector<UnitigStrand>& unitigs);
// graph_simplification.rs:315-526
void merge_linear_paths(UnitigGraph& graph, const std::vector<Sequence>& seqs);
void merge_fixed_sets(const UnitigGraph& graph, const std::vector<Sequence>& seqs, std::unordered_set<uint32_t>& fixed_starts,
                      std::unordered_set<uint32_t>& fixed_ends);           // the two sets merge_linear_paths works from (:330-331)
std::string merge_unitig_seqs(const std::vector<UnitigStrand>& path);      // :490-500

// cluster.rs:132-176: all-against-all contig distances from the unitig sets of the paths, as the PHYLIP-style matrix file
std::string pairwise_distance_matrix(const UnitigGraph& graph, const std::vector<Sequence>& sequences);

// decompress.rs:83-114
void save_original_seqs_to_dir(const std::string& out_dir, const UnitigGraph& g, const std::vector<Sequence>& seqs);

}  // namespace orc
