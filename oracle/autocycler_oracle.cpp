// ORACLE — TEST INFRASTRUCTURE ONLY (see autocycler_oracle.hpp for the rules and the pinning statement).
// CPU restatement of rrwick/Autocycler v0.6.1 `compress` (+ the GFA loader / decompress used by the
// reference's own end-to-end invariants).  Citations are file:line under the reference's src/.
#include "autocycler_oracle.hpp"

#include <dirent.h>
#include <sys/stat.h>
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <cassert>
#include <cctype>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>
#include <thread>

namespace orc {

// ---------------------------------------------------------------------------------------------
// misc.rs
// ---------------------------------------------------------------------------------------------
void quit_with_error(const std::string& text) { throw OracleError{text}; }   // misc.rs:137-141 (test cfg: panic)

#define ORC_ASSERT(cond, msg) do { if (!(cond)) throw OracleError{std::string("assertion failed: ") + msg}; } while (0)

static char complement_base(char b) {   // misc.rs:324-333
    switch (b) { case 'A': return 'T'; case 'T': return 'A'; case 'G': return 'C'; case 'C': return 'G';
                 case '.': return '.'; default: return 'N'; }
}

std::string reverse_complement(const std::string& s) {   // misc.rs:336-342
    std::string r(s.size(), 'N');
    for (size_t i = 0; i < s.size(); ++i) r[i] = complement_base(s[s.size() - 1 - i]);
    return r;
}

static bool ends_with(const std::string& s, const std::string& suf) {
    return s.size() >= suf.size() && s.compare(s.size() - suf.size(), suf.size(), suf) == 0;
}

// Rust Path::extension / file_stem on the final component: split at the LAST '.', except that a
// name starting with '.' and having no other '.' has no extension.
static void split_ext(const std::string& name, std::string& stem, std::string& ext) {
    size_t dot = name.rfind('.');
    if (dot == std::string::npos || dot == 0) { stem = name; ext.clear(); return; }
    stem = name.substr(0, dot); ext = name.substr(dot + 1);
}

static bool is_regular_file(const std::string& p) { struct stat st; return stat(p.c_str(), &st) == 0 && S_ISREG(st.st_mode); }
static bool is_dir(const std::string& p) { struct stat st; return stat(p.c_str(), &st) == 0 && S_ISDIR(st.st_mode); }

static bool is_assembly_file(const std::string& path) {   // misc.rs:86-95, incl. the &&/|| precedence quirk
    if (!is_regular_file(path)) return false;
    size_t slash = path.rfind('/');
    std::string name = slash == std::string::npos ? path : path.substr(slash + 1), stem, ext;
    split_ext(name, stem, ext);
    return ext == "fasta" || ext == "fna" || ext == "fa" ||
           ((ext == "gz" && ends_with(stem, ".fasta")) || ends_with(stem, ".fna") || ends_with(stem, ".fa"));
}

std::vector<std::string> find_all_assemblies(const std::string& in_dir) {   // misc.rs:64-83
    DIR* d = opendir(in_dir.c_str());
    if (!d) quit_with_error("unable to read directory " + in_dir);
    std::vector<std::string> all;
    while (dirent* e = readdir(d)) {
        std::string n = e->d_name;
        if (n == "." || n == "..") continue;
        std::string p = in_dir + (ends_with(in_dir, "/") ? "" : "/") + n;
        if (is_assembly_file(p)) all.push_back(p);
    }
    closedir(d);
    std::sort(all.begin(), all.end());   // PathBuf ordering is component-wise; same dir => by file name bytes
    if (all.empty()) quit_with_error("no assemblies found in " + in_dir);
    return all;
}

static bool read_whole_file(const std::string& filename, std::string& out, bool* gz) {
    FILE* f = fopen(filename.c_str(), "rb");
    if (!f) return false;
    unsigned char magic[2]; size_t n = fread(magic, 1, 2, f); fclose(f);
    *gz = (n == 2 && magic[0] == 0x1f && magic[1] == 0x8b);   // misc.rs:233-245
    out.clear();
    if (*gz) {   // MultiGzDecoder: gzread walks concatenated members
        gzFile g = gzopen(filename.c_str(), "rb");
        if (!g) return false;
        char buf[1 << 16]; int r;
        while ((r = gzread(g, buf, sizeof buf)) > 0) out.append(buf, r);
        gzclose(g);
        return r == 0;
    }
    std::ifstream in(filename, std::ios::binary);
    if (!in) return false;
    std::ostringstream ss; ss << in.rdbuf(); out = ss.str();
    return true;
}

static std::vector<std::string> split_whitespace(const std::string& s) {
    std::vector<std::string> v; size_t i = 0;
    while (i < s.size()) {
        while (i < s.size() && isspace((unsigned char)s[i])) ++i;
        size_t j = i;
        while (j < s.size() && !isspace((unsigned char)s[j])) ++j;
        if (j > i) v.push_back(s.substr(i, j - i));
        i = j;
    }
    return v;
}

std::vector<std::tuple<std::string, std::string, std::string>> load_fasta(const std::string& filename) {
    // misc.rs:144-159 (load_fasta), :248-321 (the two loaders are the same state machine), :174-194 (checks)
    struct stat st;
    if (stat(filename.c_str(), &st) == 0 && st.st_size == 0) quit_with_error(filename + " is an empty file");
    std::string data; bool gz = false;
    if (!read_whole_file(filename, data, &gz)) quit_with_error("unable to load " + filename);
    std::vector<std::tuple<std::string, std::string, std::string>> fasta_seqs;
    std::string name, header, sequence;
    auto flush = [&]() {
        for (auto& c : sequence) c = (char)toupper((unsigned char)c);   // make_ascii_uppercase
        fasta_seqs.emplace_back(name, header, sequence);
        sequence.clear();
    };
    size_t i = 0;
    while (i < data.size()) {   // BufRead::lines: split on '\n', strip one trailing '\r'
        size_t j = data.find('\n', i);
        if (j == std::string::npos) j = data.size();
        std::string text = data.substr(i, j - i);
        i = j + 1;
        if (!text.empty() && text.back() == '\r') text.pop_back();
        if (text.empty()) continue;
        if (text[0] == '>') {
            if (!name.empty()) flush();
            header = text.substr(1);
            auto pieces = split_whitespace(header);
            if (pieces.empty()) quit_with_error(filename + " is not correctly formatted");
            name = pieces[0];
        } else {
            if (name.empty()) quit_with_error(filename + " is not correctly formatted");
            sequence += text;
        }
    }
    if (!name.empty()) flush();
    if (fasta_seqs.empty()) quit_with_error(filename + " contains no sequences");
    for (auto& t : fasta_seqs) {
        if (std::get<0>(t).empty()) quit_with_error(filename + " has an unnamed sequence");
        if (std::get<2>(t).empty()) quit_with_error(filename + " has an empty sequence");
    }
    std::unordered_set<std::string> names;
    for (auto& t : fasta_seqs)
        if (!names.insert(std::get<0>(t)).second)
            quit_with_error(filename + " has a duplicate name: " + std::get<0>(t));
    return fasta_seqs;
}

// ---------------------------------------------------------------------------------------------
// position.rs, sequence.rs
// ---------------------------------------------------------------------------------------------
std::string Position::to_string() const {   // position.rs:54-58
    return std::to_string(seq_id()) + (strand() ? "+" : "-") + std::to_string(pos);
}

Sequence Sequence::new_with_seq(size_t id, std::string seq, std::string filename, std::string contig_header,
                                size_t length, uint32_t half_k) {   // sequence.rs:31-59
    for (char c : seq)
        if (!(c == 'A' || c == 'C' || c == 'G' || c == 'T')) quit_with_error(filename + " contains non-ACGT characters");
    Sequence s;
    s.forward_seq = std::string(half_k, '.') + seq + std::string(half_k, '.');
    s.reverse_seq = reverse_complement(s.forward_seq);
    s.id = (uint16_t)id; s.filename = std::move(filename); s.contig_header = std::move(contig_header);
    s.length = length; s.cluster = 0;
    return s;
}

Sequence Sequence::new_without_seq(uint16_t id, std::string filename, std::string contig_header, size_t length,
                                   uint16_t cluster) {   // sequence.rs:61-75
    Sequence s; s.id = id; s.filename = std::move(filename); s.contig_header = std::move(contig_header);
    s.length = length; s.cluster = cluster; return s;
}

static std::string lower(std::string s) { for (auto& c : s) c = (char)tolower((unsigned char)c); return s; }
std::string Sequence::contig_name() const {   // misc.rs:462-465 up_to_first_space
    size_t p = contig_header.find(' '); return p == std::string::npos ? contig_header : contig_header.substr(0, p);
}
std::string Sequence::contig_description() const {   // misc.rs:467-471 after_first_space
    size_t p = contig_header.find(' '); return p == std::string::npos ? std::string() : contig_header.substr(p + 1);
}
bool Sequence::is_ignored() const { return lower(contig_header).find("autocycler_ignore") != std::string::npos; }
bool Sequence::is_trusted() const { return lower(contig_header).find("autocycler_trusted") != std::string::npos; }
static size_t header_weight(const std::string& contig_header, const std::string& key) {   // sequence.rs:96-108
    const std::string low = lower(contig_header);
    for (const std::string& token : split_whitespace(low))
        if (token.compare(0, key.size(), key) == 0) {
            const std::string v = token.substr(key.size());
            if (!v.empty() && v.find_first_not_of("0123456789", v[0] == '+' ? 1 : 0) == std::string::npos && v != "+") return (size_t)strtoull(v.c_str(), nullptr, 10);
        }
    return 1;
}
size_t Sequence::cluster_weight() const { return header_weight(contig_header, "autocycler_cluster_weight="); }
size_t Sequence::consensus_weight() const { return header_weight(contig_header, "autocycler_consensus_weight="); }
std::string Sequence::display() const {   // sequence.rs:112-135
    std::vector<std::string> extras;
    if (is_trusted()) extras.push_back("trusted");
    if (is_ignored()) extras.push_back("ignored");
    if (cluster_weight() != 1) extras.push_back("cluster weight = " + std::to_string(cluster_weight()));
    if (consensus_weight() != 1) extras.push_back("consensus weight = " + std::to_string(consensus_weight()));
    std::string s = filename + " " + contig_name() + " (" + std::to_string(length) + " bp)";
    if (!extras.empty()) { s += " ["; for (size_t i = 0; i < extras.size(); ++i) { if (i) s += ", "; s += extras[i]; } s += "]"; }
    return s;
}

// ---------------------------------------------------------------------------------------------
// compress.rs: load_sequences, end repair
// ---------------------------------------------------------------------------------------------
std::string find_best_match(const std::vector<std::string>& matches) {   // compress.rs:239-270
    ORC_ASSERT(!matches.empty(), "There should be at least one match");
    std::unordered_map<std::string, std::pair<size_t, size_t>> counts;   // (freq, dots)
    for (auto& m : matches) {
        auto& e = counts[m];
        e.first += 1;
        e.second = (size_t)std::count(m.begin(), m.end(), '.');
    }
    const std::string* best = nullptr;
    for (auto& m : matches) {   // Iterator::min_by keeps the FIRST minimum; ties are equal strings anyway
        if (!best) { best = &m; continue; }
        auto& a = counts[m]; auto& b = counts[*best];
        bool less;
        if (a.second != b.second) less = a.second < b.second;          // fewer dots
        else if (a.first != b.first) less = a.first > b.first;         // higher frequency
        else less = m < *best;                                         // alphabetical
        if (less) best = &m;
    }
    return *best;
}

// Leftmost, non-overlapping matches (regex `find_iter`) of a pattern whose bytes are literals or the
// wildcard '.', which matches any byte (compress.rs:212-229).
static void find_iter(const std::string& pat, const std::string& hay, std::vector<std::string>& out) {
    const size_t m = pat.size(), n = hay.size();
    if (m == 0 || n < m) return;
    size_t lit = 0; while (lit < m && pat[lit] == '.') ++lit;     // first literal index
    size_t pos = 0;
    while (pos + m <= n) {
        bool ok = true;
        if (lit < m) {
            // jump to the next candidate using the first literal byte
            const void* p = memchr(hay.data() + pos + lit, pat[lit], n - m - pos + 1);
            if (!p) return;
            pos = (const char*)p - hay.data() - lit;
            for (size_t i = lit; i < m; ++i) if (pat[i] != '.' && pat[i] != hay[pos + i]) { ok = false; break; }
        }
        if (ok) { out.emplace_back(hay, pos, m); pos += m; } else { pos += 1; }
    }
}

void sequence_end_repair(std::vector<Sequence>& sequences, uint32_t k_size, int threads) {   // compress.rs:202-236
    const size_t overlap = k_size - 1;
    if (overlap == 0) return;   // k=1: empty regex, empty best match, splice is a no-op
    std::vector<std::string> all_seqs;
    for (auto& s : sequences) { all_seqs.push_back(s.forward_seq); all_seqs.push_back(s.reverse_seq); }
    std::atomic<size_t> next{0};
    auto work = [&]() {
        for (;;) {
            size_t i = next.fetch_add(1);
            if (i >= sequences.size()) return;
            Sequence& seq = sequences[i];
            std::string start = seq.forward_seq.substr(0, overlap);
            std::string end = seq.forward_seq.substr(seq.forward_seq.size() - overlap);
            std::vector<std::string> all_matches;
            for (auto& s : all_seqs) find_iter(start, s, all_matches);
            std::string best = find_best_match(all_matches);
            seq.forward_seq.replace(0, overlap, best);
            all_matches.clear();
            for (auto& s : all_seqs) find_iter(end, s, all_matches);
            best = find_best_match(all_matches);
            seq.forward_seq.replace(seq.forward_seq.size() - overlap, overlap, best);
            seq.reverse_seq = reverse_complement(seq.forward_seq);
        }
    };
    int nt = std::max(1, std::min<int>(threads, (int)sequences.size()));
    std::vector<std::thread> pool;
    for (int t = 1; t < nt; ++t) pool.emplace_back(work);
    work();
    for (auto& t : pool) t.join();
}

std::pair<std::vector<Sequence>, size_t> load_sequences(const std::string& assemblies_dir, uint32_t k_size,
                                                        InputAssemblyMetrics& metrics, uint32_t max_contigs,
                                                        int threads, bool verbose) {   // compress.rs:98-133
    auto assemblies = find_all_assemblies(assemblies_dir);
    const uint32_t half_k = k_size / 2;
    size_t seq_id = 0;
    std::vector<Sequence> sequences;
    for (auto& assembly : assemblies) {
        InputAssemblyDetails details; details.filename = assembly;
        for (auto& rec : load_fasta(assembly)) {
            const std::string& header = std::get<1>(rec);
            const std::string& seq = std::get<2>(rec);
            size_t seq_len = seq.size();
            if (seq_len < k_size) continue;
            seq_id += 1;
            if (seq_id > 32767) quit_with_error("no more than 32767 input sequences are allowed");
            std::string contig_header;
            for (auto& w : split_whitespace(header)) { if (!contig_header.empty()) contig_header += ' '; contig_header += w; }
            size_t slash = assembly.rfind('/');
            std::string filename = slash == std::string::npos ? assembly : assembly.substr(slash + 1);
            Sequence s = Sequence::new_with_seq(seq_id, seq, filename, contig_header, seq_len, half_k);
            if (verbose) fprintf(stderr, " %3zu: %s\n", seq_id, s.display().c_str());
            details.contigs.push_back({s.contig_name(), s.contig_description(), (uint64_t)s.length});
            if (!s.is_ignored()) sequences.push_back(std::move(s));
        }
        metrics.input_assembly_details.push_back(std::move(details));
    }
    // check_sequence_count, compress.rs:84-95
    double sequence_count = (double)sequences.size();
    if (sequence_count == 0.0) quit_with_error("no sequences found in input assemblies");
    double mean = sequence_count / (double)assemblies.size();
    if (mean > (double)max_contigs) {
        char buf[256];
        snprintf(buf, sizeof buf, "the mean number of contigs per input assembly (%.1f) exceeds the allowed threshold (%u). "
                 "Are your input assemblies fragmented or contaminated?", mean, max_contigs);
        quit_with_error(buf);
    }
    sequence_end_repair(sequences, k_size, threads);
    return {std::move(sequences), assemblies.size()};
}

// ---------------------------------------------------------------------------------------------
// kmer_graph.rs
// ---------------------------------------------------------------------------------------------
static const char ALPHABET[5] = {'.', 'A', 'C', 'G', 'T'};   // kmer_graph.rs:23

std::string Kmer::display() const {   // kmer_graph.rs:63-70
    std::string s = seq() + ":";
    for (size_t i = 0; i < positions.size(); ++i) { if (i) s += ","; s += positions[i].to_string(); }
    return s;
}

uint64_t KmerGraph::hash(const char* p) const {   // FxHash-style word mixing; iteration order is never used
    uint64_t h = 0; size_t n = k_size, i = 0;
    for (; i + 8 <= n; i += 8) { uint64_t w; memcpy(&w, p + i, 8); h = ((h << 5 | h >> 59) ^ w) * 0x517cc1b727220a95ULL; }
    if (i < n) { uint64_t w = 0; memcpy(&w, p + i, n - i); h = ((h << 5 | h >> 59) ^ w) * 0x517cc1b727220a95ULL; }
    return h ^ (h >> 29);
}

void KmerGraph::grow() {
    size_t cap = table.empty() ? (1u << 16) : table.size() * 2;
    table.assign(cap, 0); mask = cap - 1;
    for (size_t i = 0; i < kmers.size(); ++i) {
        size_t s = hash(kmers[i].pointer) & mask;
        while (table[s]) s = (s + 1) & mask;
        table[s] = (uint32_t)(i + 1);
    }
}

Kmer* KmerGraph::get(const char* key) {
    if (table.empty()) return nullptr;
    size_t s = hash(key) & mask;
    while (table[s]) {
        Kmer& k = kmers[table[s] - 1];
        if (memcmp(k.pointer, key, k_size) == 0) return &k;
        s = (s + 1) & mask;
    }
    return nullptr;
}

Kmer* KmerGraph::entry(const char* key, size_t assembly_count, bool* created) {
    if ((kmers.size() + 1) * 2 > table.size()) grow();
    size_t s = hash(key) & mask;
    while (table[s]) {
        Kmer& k = kmers[table[s] - 1];
        if (memcmp(k.pointer, key, k_size) == 0) { *created = false; return &k; }
        s = (s + 1) & mask;
    }
    kmers.emplace_back();
    Kmer& k = kmers.back();
    k.pointer = key; k.length = k_size; k.positions.reserve(assembly_count);   // kmer_graph.rs:36-42
    table[s] = (uint32_t)kmers.size();
    *created = true;
    return &k;
}

void KmerGraph::add_sequences(const std::vector<Sequence>& seqs, size_t assembly_count) {   // kmer_graph.rs:86-90
    for (auto& s : seqs) add_sequence(s, assembly_count);
}

void KmerGraph::add_sequence(const Sequence& seq, size_t assembly_count) {   // kmer_graph.rs:92-134
    const size_t k = k_size, half_k = k_size / 2, two_half_k = half_k + half_k;
    const char* forward_raw = seq.forward_seq.data();
    const char* reverse_raw = seq.reverse_seq.data();
    for (size_t forward_start = 0; forward_start < seq.length; ++forward_start) {
        size_t forward_end = forward_start + k;
        size_t reverse_start = seq.length + two_half_k - forward_end;
        bool created;
        entry(forward_raw + forward_start, assembly_count, &created)->positions.emplace_back(seq.id, strand::FORWARD, forward_start);
        entry(reverse_raw + reverse_start, assembly_count, &created)->positions.emplace_back(seq.id, strand::REVERSE, reverse_start);
    }
}

std::vector<Kmer*> KmerGraph::next_kmers(const char* kmer) {   // kmer_graph.rs:136-150
    std::vector<Kmer*> out;
    std::string next(kmer + 1, k_size - 1); next.push_back('N');
    for (char base : ALPHABET) { next.back() = base; if (Kmer* k = get(next.data())) out.push_back(k); }
    return out;
}

std::vector<Kmer*> KmerGraph::prev_kmers(const char* kmer) {   // kmer_graph.rs:152-166
    std::vector<Kmer*> out;
    std::string prev(1, 'N'); prev.append(kmer, k_size - 1);
    for (char base : ALPHABET) { prev[0] = base; if (Kmer* k = get(prev.data())) out.push_back(k); }
    return out;
}

std::vector<Kmer*> KmerGraph::iterate_kmers() {   // kmer_graph.rs:168-173: keys sorted bytewise
    std::vector<Kmer*> v; v.reserve(kmers.size());
    for (auto& k : kmers) v.push_back(&k);
    const size_t k = k_size;
    std::sort(v.begin(), v.end(), [k](const Kmer* a, const Kmer* b) { return memcmp(a->pointer, b->pointer, k) < 0; });
    return v;
}

Kmer* KmerGraph::reverse(const Kmer* kmer) {   // kmer_graph.rs:175-181
    std::string rc = reverse_complement(std::string(kmer->pointer, k_size));
    Kmer* r = get(rc.data());
    ORC_ASSERT(r != nullptr, "reverse-complement k-mer must exist");
    return r;
}

// ---------------------------------------------------------------------------------------------
// unitig.rs
// ---------------------------------------------------------------------------------------------
uint32_t UnitigStrand::number() const { return unitig->number; }

Unitig Unitig::from_kmers(uint32_t number, Kmer* f, Kmer* r) {   // unitig.rs:48-60
    Unitig u; u.number = number; u.forward_kmers.push_back(f); u.reverse_kmers.push_back(r); return u;
}

static std::vector<std::string> split_tab(const std::string& s) {
    std::vector<std::string> parts; size_t i = 0;
    for (;;) { size_t j = s.find('\t', i); if (j == std::string::npos) { parts.push_back(s.substr(i)); break; }
               parts.push_back(s.substr(i, j - i)); i = j + 1; }
    return parts;
}

Unitig Unitig::from_segment_line(const std::string& line) {   // unitig.rs:62-91
    auto parts = split_tab(line);
    if (parts.size() < 3) quit_with_error("Segment line does not have enough parts.");
    Unitig u;
    char* endp = nullptr;
    unsigned long num = strtoul(parts[1].c_str(), &endp, 10);
    if (parts[1].empty() || *endp) quit_with_error("Unable to parse unitig number.");
    u.number = (uint32_t)num;
    u.forward_seq = parts[2];
    u.reverse_seq = reverse_complement(u.forward_seq);
    bool found = false;
    for (auto& p : parts)
        if (p.rfind("DP:f:", 0) == 0) {
            char* e = nullptr; double d = strtod(p.c_str() + 5, &e);
            if (e != p.c_str() + 5 && *e == 0) { u.depth = d; found = true; }
            break;   // Iterator::find stops at the first DP:f: part
        }
    if (!found) quit_with_error("Could not find a depth tag (e.g. DP:f:10.00) in the GFA segment line.");
    auto has = [&](const char* tag) { for (auto& p : parts) if (p == tag) return true; return false; };   // unitig.rs:78-86
    u.unitig_type = has("CL:Z:steelblue") ? UnitigType::Consentig : has("CL:Z:forestgreen") ? UnitigType::Anchor
                  : has("CL:Z:pink") ? UnitigType::Bridge : UnitigType::Other;
    return u;
}

void Unitig::add_kmer_to_end(Kmer* f, Kmer* r) { forward_kmers.push_back(f); reverse_kmers.push_front(r); }     // unitig.rs:102-105
void Unitig::add_kmer_to_start(Kmer* f, Kmer* r) { forward_kmers.push_front(f); reverse_kmers.push_back(r); }   // unitig.rs:107-110

void Unitig::simplify_seqs() {   // unitig.rs:112-155
    if (!forward_kmers.empty()) {
        forward_seq = forward_kmers.front()->seq();
        for (size_t i = 1; i < forward_kmers.size(); ++i) forward_seq.push_back(forward_kmers[i]->pointer[forward_kmers[i]->length - 1]);
    }
    if (!reverse_kmers.empty()) {
        reverse_seq = reverse_kmers.front()->seq();
        for (size_t i = 1; i < reverse_kmers.size(); ++i) reverse_seq.push_back(reverse_kmers[i]->pointer[reverse_kmers[i]->length - 1]);
    }
    if (!forward_kmers.empty()) forward_positions = forward_kmers.front()->positions;
    if (!reverse_kmers.empty()) reverse_positions = reverse_kmers.front()->positions;
    double fsum = 0.0, rsum = 0.0;
    for (auto* k : forward_kmers) fsum += (double)k->depth();
    for (auto* k : reverse_kmers) rsum += (double)k->depth();
    double favg = fsum / (double)forward_kmers.size(), ravg = rsum / (double)reverse_kmers.size();
    ORC_ASSERT(favg == ravg, "forward and reverse mean depth differ");
    depth = favg;
    forward_kmers.clear(); reverse_kmers.clear();
}

void Unitig::trim_overlaps(size_t k_size) {   // unitig.rs:157-165
    size_t overlap = k_size / 2;
    ORC_ASSERT(forward_seq.size() >= k_size, "unitig shorter than k");
    forward_seq = forward_seq.substr(overlap);
    reverse_seq = reverse_seq.substr(0, reverse_seq.size() - overlap);
    forward_seq = forward_seq.substr(0, forward_seq.size() - overlap);
    reverse_seq = reverse_seq.substr(overlap);
    ORC_ASSERT(!forward_seq.empty(), "empty unitig after trim");
}

std::string Unitig::gfa_segment_line() const {   // unitig.rs:167-181 with use_other_colour=false
    char dp[64]; snprintf(dp, sizeof dp, "%.2f", depth);
    const char* colour = unitig_type == UnitigType::Consentig ? "\tCL:Z:steelblue" : unitig_type == UnitigType::Anchor ? "\tCL:Z:forestgreen"
                       : unitig_type == UnitigType::Bridge ? "\tCL:Z:pink" : "";
    return "S\t" + std::to_string(number) + "\t" + forward_seq + "\tDP:f:" + dp + colour;
}

void Unitig::remove_seq_from_start(size_t amount) {   // unitig.rs:216-223
    for (auto& p : forward_positions) p.pos += (uint32_t)amount;
    ORC_ASSERT(amount <= forward_seq.size(), "remove_seq_from_start amount");
    forward_seq.erase(0, amount);
    reverse_seq.resize(reverse_seq.size() - amount);
}
void Unitig::remove_seq_from_end(size_t amount) {   // unitig.rs:225-232
    for (auto& p : reverse_positions) p.pos += (uint32_t)amount;
    ORC_ASSERT(amount <= forward_seq.size(), "remove_seq_from_end amount");
    forward_seq.resize(reverse_seq.size() - amount);
    reverse_seq.erase(0, amount);
}
void Unitig::add_seq_to_start(const std::string& seq) {   // unitig.rs:234-240
    for (auto& p : forward_positions) p.pos -= (uint32_t)seq.size();
    forward_seq.insert(0, seq);
    reverse_seq = reverse_complement(forward_seq);
}
void Unitig::add_seq_to_end(const std::string& seq) {   // unitig.rs:242-248
    for (auto& p : reverse_positions) p.pos -= (uint32_t)seq.size();
    forward_seq += seq;
    reverse_seq = reverse_complement(forward_seq);
}

// ---------------------------------------------------------------------------------------------
// unitig_graph.rs
// ---------------------------------------------------------------------------------------------
UnitigGraph UnitigGraph::from_kmer_graph(KmerGraph& kg) {   // unitig_graph.rs:36-48
    UnitigGraph g; g.k_size = kg.k_size;
    g.build_unitigs_from_kmer_graph(kg);
    g.simplify_seqs();
    g.create_links();
    g.trim_overlaps();
    g.renumber_unitigs();
    g.check_links();
    return g;
}

void UnitigGraph::build_unitig_index() {   // unitig_graph.rs:76-78
    unitig_index.clear();
    for (auto& u : unitigs) unitig_index[u->number] = u.get();
}

void UnitigGraph::build_unitigs_from_kmer_graph(KmerGraph& kg) {   // unitig_graph.rs:176-226
    uint32_t unitig_number = 0;
    for (Kmer* forward_kmer : kg.iterate_kmers()) {
        if (forward_kmer->seen) continue;
        Kmer* reverse_kmer = kg.reverse(forward_kmer);
        unitig_number += 1;
        auto unitig = std::make_unique<Unitig>(Unitig::from_kmers(unitig_number, forward_kmer, reverse_kmer));
        forward_kmer->seen = true; reverse_kmer->seen = true;

        // extend forward
        Kmer* for_k = forward_kmer; Kmer* rev_k = reverse_kmer;
        for (;;) {
            if (rev_k->first_position()) break;
            auto next = kg.next_kmers(for_k->pointer);
            if (next.size() != 1) break;
            for_k = next[0];
            if (for_k->seen) break;
            auto prev = kg.prev_kmers(for_k->pointer);
            if (prev.size() != 1) break;
            rev_k = kg.reverse(for_k);
            if (for_k->first_position()) break;
            unitig->add_kmer_to_end(for_k, rev_k);
            for_k->seen = true; rev_k->seen = true;
        }
        // extend backward
        for_k = forward_kmer;
        for (;;) {
            if (for_k->first_position()) break;
            auto prev = kg.prev_kmers(for_k->pointer);
            if (prev.size() != 1) break;
            for_k = prev[0];
            if (for_k->seen) break;
            auto next = kg.next_kmers(for_k->pointer);
            if (next.size() != 1) break;
            rev_k = kg.reverse(for_k);
            if (rev_k->first_position()) break;
            unitig->add_kmer_to_start(for_k, rev_k);
            for_k->seen = true; rev_k->seen = true;
        }
        unitigs.push_back(std::move(unitig));
    }
}

void UnitigGraph::simplify_seqs() { for (auto& u : unitigs) u->simplify_seqs(); }   // unitig_graph.rs:228-232

void UnitigGraph::create_links() {   // unitig_graph.rs:234-287
    const size_t piece_len = k_size - 1;
    std::unordered_map<std::string, std::vector<size_t>> forward_starts, reverse_starts;
    for (size_t i = 0; i < unitigs.size(); ++i) {
        forward_starts[unitigs[i]->forward_seq.substr(0, piece_len)].push_back(i);
        reverse_starts[unitigs[i]->reverse_seq.substr(0, piece_len)].push_back(i);
    }
    for (size_t i = 0; i < unitigs.size(); ++i) {
        Unitig* a = unitigs[i].get();
        std::string ending_forward = a->forward_seq.substr(a->forward_seq.size() - piece_len);
        std::string ending_reverse = a->reverse_seq.substr(a->reverse_seq.size() - piece_len);
        auto it = forward_starts.find(ending_forward);
        if (it != forward_starts.end())
            for (size_t j : it->second) {
                Unitig* b = unitigs[j].get();
                a->forward_next.push_back({b, strand::FORWARD});   // a+ -> b+
                b->forward_prev.push_back({a, strand::FORWARD});
                b->reverse_next.push_back({a, strand::REVERSE});   // b- -> a-
                a->reverse_prev.push_back({b, strand::REVERSE});
            }
        it = reverse_starts.find(ending_forward);
        if (it != reverse_starts.end())
            for (size_t j : it->second) {
                Unitig* b = unitigs[j].get();
                a->forward_next.push_back({b, strand::REVERSE});   // a+ -> b-
                b->reverse_prev.push_back({a, strand::FORWARD});
            }
        it = forward_starts.find(ending_reverse);
        if (it != forward_starts.end())
            for (size_t j : it->second) {
                Unitig* b = unitigs[j].get();
                a->reverse_next.push_back({b, strand::FORWARD});   // a- -> b+
                b->forward_prev.push_back({a, strand::REVERSE});
            }
    }
}

void UnitigGraph::trim_overlaps() { for (auto& u : unitigs) u->trim_overlaps(k_size); }   // unitig_graph.rs:289-293

void UnitigGraph::renumber_unitigs() {   // unitig_graph.rs:295-315 (slice::sort_by is stable)
    std::stable_sort(unitigs.begin(), unitigs.end(), [](const std::unique_ptr<Unitig>& a, const std::unique_ptr<Unitig>& b) {
        if (a->length() != b->length()) return a->length() > b->length();
        int c = a->forward_seq.compare(b->forward_seq);
        if (c != 0) return c < 0;
        return a->depth > b->depth;
    });
    for (size_t i = 0; i < unitigs.size(); ++i) unitigs[i]->number = (uint32_t)(i + 1);
    build_unitig_index();
}

std::string UnitigGraph::gfa_text(const std::vector<Sequence>& sequences) const {   // unitig_graph.rs:317-360
    std::string out = "H\tVN:Z:1.0\tKM:i:" + std::to_string(k_size) + "\n";
    for (auto& u : unitigs) { out += u->gfa_segment_line(); out += '\n'; }
    for (auto& a : unitigs) {   // get_links_for_gfa, :333-350
        for (auto& b : a->forward_next)
            out += "L\t" + std::to_string(a->number) + "\t+\t" + std::to_string(b.number()) + "\t" + (b.strand ? "+" : "-") + "\t0M\n";
        for (auto& b : a->reverse_next)
            out += "L\t" + std::to_string(a->number) + "\t-\t" + std::to_string(b.number()) + "\t" + (b.strand ? "+" : "-") + "\t0M\n";
    }
    for (auto& s : sequences) {   // get_gfa_path_line, :352-360
        auto path = get_unitig_path_for_sequence(s);
        std::string path_str;
        for (size_t i = 0; i < path.size(); ++i) {
            if (i) path_str += ',';
            path_str += std::to_string(path[i].first); path_str += path[i].second ? '+' : '-';
        }
        out += "P\t" + std::to_string(s.id) + "\t" + path_str + "\t*\tLN:i:" + std::to_string(s.length) +
               "\tFN:Z:" + s.filename + "\tHD:Z:" + s.contig_header;
        if (s.cluster > 0) out += "\tCL:i:" + std::to_string(s.cluster);
        out += '\n';
    }
    return out;
}

static std::vector<std::pair<uint32_t, bool>> parse_unitig_path(const std::string& s) {   // unitig_graph.rs (parse_unitig_path)
    std::vector<std::pair<uint32_t, bool>> path;
    size_t i = 0;
    while (i < s.size()) {
        size_t j = s.find(',', i); if (j == std::string::npos) j = s.size();
        std::string tok = s.substr(i, j - i);
        if (!tok.empty()) {
            bool st = tok.back() == '+';
            if (tok.back() != '+' && tok.back() != '-') quit_with_error("Invalid path strand");
            path.emplace_back((uint32_t)strtoul(tok.substr(0, tok.size() - 1).c_str(), nullptr, 10), st);
        }
        i = j + 1;
    }
    return path;
}

std::pair<UnitigGraph, std::vector<Sequence>> UnitigGraph::from_gfa_lines(const std::vector<std::string>& lines) {
    // unitig_graph.rs:55-174
    UnitigGraph g;
    std::vector<const std::string*> link_lines, path_lines;
    for (auto& raw : lines) {
        std::string line = raw;
        while (!line.empty() && line.back() == '\n') line.pop_back();
        auto parts = split_tab(line);
        if (parts[0] == "H") {
            for (auto& p : parts) if (p.rfind("KM:i:", 0) == 0) { g.k_size = (uint32_t)strtoul(p.c_str() + 5, nullptr, 10); break; }
        } else if (parts[0] == "S") g.unitigs.push_back(std::make_unique<Unitig>(Unitig::from_segment_line(line)));
        else if (parts[0] == "L") link_lines.push_back(&raw);
        else if (parts[0] == "P") path_lines.push_back(&raw);
    }
    g.build_unitig_index();
    for (auto* lp : link_lines) {   // build_links_from_gfa :91-115
        std::string line = *lp; while (!line.empty() && line.back() == '\n') line.pop_back();
        auto parts = split_tab(line);
        if (parts.size() < 6 || parts[5] != "0M") quit_with_error("non-zero overlap found on the GFA link line.");
        uint32_t seg1 = (uint32_t)strtoul(parts[1].c_str(), nullptr, 10), seg2 = (uint32_t)strtoul(parts[3].c_str(), nullptr, 10);
        bool s1 = parts[2] == "+", s2 = parts[4] == "+";
        auto i1 = g.unitig_index.find(seg1);
        if (i1 == g.unitig_index.end()) quit_with_error("link refers to nonexistent unitig: " + parts[1]);
        auto i2 = g.unitig_index.find(seg2);
        if (i2 == g.unitig_index.end()) quit_with_error("link refers to nonexistent unitig: " + parts[3]);
        Unitig* u1 = i1->second; Unitig* u2 = i2->second;
        if (s1) u1->forward_next.push_back({u2, s2}); else u1->reverse_next.push_back({u2, s2});
        if (s2) u2->forward_prev.push_back({u1, s1}); else u2->reverse_prev.push_back({u1, s1});
    }
    std::vector<Sequence> sequences;
    for (auto* pp : path_lines) {   // build_paths_from_gfa :117-174
        std::string line = *pp; while (!line.empty() && line.back() == '\n') line.pop_back();
        auto parts = split_tab(line);
        uint16_t seq_id = (uint16_t)strtoul(parts[1].c_str(), nullptr, 10);
        bool has_len = false, has_fn = false, has_hd = false; uint32_t length = 0; std::string filename, header; uint16_t cluster = 0;
        for (size_t i = 2; i < parts.size(); ++i) {
            auto& p = parts[i];
            if (p.rfind("LN:i:", 0) == 0) { length = (uint32_t)strtoul(p.c_str() + 5, nullptr, 10); has_len = true; }
            else if (p.rfind("FN:Z:", 0) == 0) { filename = p.substr(5); has_fn = true; }
            else if (p.rfind("HD:Z:", 0) == 0) { header = p.substr(5); has_hd = true; }
            else if (p.rfind("CL:i:", 0) == 0) cluster = (uint16_t)strtoul(p.c_str() + 5, nullptr, 10);
        }
        if (!has_len || !has_fn || !has_hd) quit_with_error("missing required tag in GFA path line.");
        auto forward_path = parse_unitig_path(parts[2]);
        std::vector<std::pair<uint32_t, bool>> reverse_path(forward_path.rbegin(), forward_path.rend());
        for (auto& e : reverse_path) e.second = !e.second;
        auto add_positions = [&](const std::vector<std::pair<uint32_t, bool>>& path, bool path_strand) {
            uint32_t pos = 0;
            for (auto& e : path) {
                auto it = g.unitig_index.find(e.first);
                if (it == g.unitig_index.end()) quit_with_error("unitig " + std::to_string(e.first) + " not found in unitig index");
                Unitig* u = it->second;
                (e.second ? u->forward_positions : u->reverse_positions).emplace_back(seq_id, path_strand, pos);
                pos += u->length();
            }
            ORC_ASSERT(pos == length, "Position calculation mismatch");
        };
        add_positions(forward_path, strand::FORWARD);
        add_positions(reverse_path, strand::REVERSE);
        sequences.push_back(Sequence::new_without_seq(seq_id, filename, header, length, cluster));
    }
    g.check_links();
    return {std::move(g), std::move(sequences)};
}

UnitigStrand UnitigGraph::find_starting_unitig(uint16_t seq_id) const {   // unitig_graph.rs:402-421
    std::vector<UnitigStrand> starting;
    for (auto& u : unitigs) {
        for (auto& p : u->forward_positions) if (p.seq_id() == seq_id && p.strand() && p.pos == 0) starting.push_back({u.get(), strand::FORWARD});
        for (auto& p : u->reverse_positions) if (p.seq_id() == seq_id && p.strand() && p.pos == 0) starting.push_back({u.get(), strand::REVERSE});
    }
    ORC_ASSERT(starting.size() == 1, "expected exactly one starting unitig");
    return starting[0];
}

bool UnitigGraph::get_next_unitig(uint16_t seq_id, bool seq_strand, const Unitig* u, bool strand, uint32_t pos,
                                  UnitigStrand* next_out, uint32_t* next_pos_out, PositionIndex* index) const {   // unitig_graph.rs:423-445
    uint32_t next_pos = pos + u->length();
    auto& next_edges = strand ? u->forward_next : u->reverse_next;
    auto key = [](uint16_t id, bool s, uint32_t p) { return (uint64_t)id << 33 | (uint64_t)s << 32 | p; };
    for (auto& next : next_edges) {
        auto& positions = next.strand ? next.unitig->forward_positions : next.unitig->reverse_positions;
        // The same answer as the scan below: the first edge whose list holds the position.  A walk through a run that repeats one unitig
        // (a homopolymer) looks its list up once per step, and the scan alone makes that walk quadratic in the run's length.
        if (index && positions.size() > 1024) {
            auto it = index->find(&positions);
            if (it == index->end()) {
                it = index->emplace(&positions, std::unordered_set<uint64_t>()).first;
                for (auto& p : positions) it->second.insert(key(p.seq_id(), p.strand(), p.pos));
            }
            if (it->second.count(key(seq_id, seq_strand, next_pos))) { *next_out = next; *next_pos_out = next_pos; return true; }
            continue;
        }
        for (auto& p : positions)
            if (p.seq_id() == seq_id && p.strand() == seq_strand && p.pos == next_pos) { *next_out = next; *next_pos_out = next_pos; return true; }
    }
    return false;
}

std::vector<std::pair<uint32_t, bool>> UnitigGraph::get_unitig_path_for_sequence(const Sequence& seq) const {   // :447-465
    std::vector<std::pair<uint32_t, bool>> path;
    UnitigStrand u = find_starting_unitig(seq.id);
    uint32_t pos = 0;
    PositionIndex index;      // the graph does not change during the walk
    for (;;) {
        path.emplace_back(u.number(), u.strand);
        UnitigStrand next; uint32_t next_pos;
        if (!get_next_unitig(seq.id, strand::FORWARD, u.unitig, u.strand, pos, &next, &next_pos, &index)) break;
        u = next; pos = next_pos;
    }
    return path;
}

std::string UnitigGraph::reconstruct_original_sequence(const Sequence& seq) const {   // unitig_graph.rs:383-400
    std::string out;
    for (auto& e : get_unitig_path_for_sequence(seq)) out += unitig_index.at(e.first)->get_seq(e.second);
    ORC_ASSERT(out.size() == seq.length, "reconstructed sequence does not have expected length");
    return out;
}

uint64_t UnitigGraph::total_length() const { uint64_t t = 0; for (auto& u : unitigs) t += u->length(); return t; }   // :474-476

std::pair<size_t, size_t> UnitigGraph::link_count() const {   // unitig_graph.rs:478-507
    std::vector<std::pair<int64_t, int64_t>> all, one;
    auto signed_num = [](const UnitigStrand& b) { return b.strand ? (int64_t)b.number() : -(int64_t)b.number(); };
    for (auto& a : unitigs) {
        int64_t an = a->number;
        for (auto& b : a->forward_next) { int64_t bn = signed_num(b); std::pair<int64_t,int64_t> l{an, bn}, r{-bn, -an}; all.push_back(l); all.push_back(r); one.push_back(l > r ? l : r); }
        for (auto& b : a->reverse_next) { int64_t bn = signed_num(b); std::pair<int64_t,int64_t> l{-an, bn}, r{-bn, an}; all.push_back(l); all.push_back(r); one.push_back(l > r ? l : r); }
    }
    auto uniq = [](std::vector<std::pair<int64_t,int64_t>>& v) { std::sort(v.begin(), v.end()); v.erase(std::unique(v.begin(), v.end()), v.end()); return v.size(); };
    return {uniq(all), uniq(one)};
}

bool UnitigGraph::link_exists(uint32_t a, bool as, uint32_t b, bool bs) const {   // unitig_graph.rs:723-735
    auto it = unitig_index.find(a); if (it == unitig_index.end()) return false;
    for (auto& n : (as ? it->second->forward_next : it->second->reverse_next)) if (n.number() == b && n.strand == bs) return true;
    return false;
}
bool UnitigGraph::link_exists_prev(uint32_t a, bool as, uint32_t b, bool bs) const {   // unitig_graph.rs:737-750
    auto it = unitig_index.find(b); if (it == unitig_index.end()) return false;
    for (auto& p : (bs ? it->second->forward_prev : it->second->reverse_prev)) if (p.number() == a && p.strand == as) return true;
    return false;
}

void UnitigGraph::check_links() const {   // unitig_graph.rs:752-793
    auto fail = [](const char* m) { throw OracleError{m}; };
    for (auto& ap : unitigs) {
        const Unitig& a = *ap;
        auto check_next = [&](const std::vector<UnitigStrand>& v, bool a_strand) {
            for (auto& b : v) {
                if (!link_exists(a.number, a_strand, b.number(), b.strand)) fail("missing next link");
                if (!link_exists_prev(a.number, a_strand, b.number(), b.strand)) fail("missing prev link");
                if (!link_exists(b.number(), !b.strand, a.number, !a_strand)) fail("missing next link");
                if (!link_exists_prev(b.number(), !b.strand, a.number, !a_strand)) fail("missing prev link");
                if (!unitig_index.count(b.number())) fail("unitig missing from index");
            }
        };
        auto check_prev = [&](const std::vector<UnitigStrand>& v, bool a_strand) {
            for (auto& b : v) {
                if (!link_exists(b.number(), b.strand, a.number, a_strand)) fail("missing next link");
                if (!link_exists_prev(b.number(), b.strand, a.number, a_strand)) fail("missing prev link");
                if (!link_exists(a.number, !a_strand, b.number(), !b.strand)) fail("missing next link");
                if (!link_exists_prev(a.number, !a_strand, b.number(), !b.strand)) fail("missing prev link");
                if (!unitig_index.count(b.number())) fail("unitig missing from index");
            }
        };
        check_next(a.forward_next, strand::FORWARD); check_next(a.reverse_next, strand::REVERSE);
        check_prev(a.forward_prev, strand::FORWARD); check_prev(a.reverse_prev, strand::REVERSE);
    }
}

// ---------------------------------------------------------------------------------------------
// graph_simplification.rs:26-312
// ---------------------------------------------------------------------------------------------
std::vector<UnitigStrand> get_exclusive_inputs(const Unitig* unitig) {   // :233-255
    std::vector<UnitigStrand> inputs;
    for (auto& prev : unitig->forward_prev) {
        auto& next = prev.strand ? prev.unitig->forward_next : prev.unitig->reverse_next;
        bool exclusive = next.size() == 1 && next[0].strand && next[0].number() == unitig->number;
        if (!exclusive) return {};
        inputs.push_back(prev);
    }
    for (auto& inp : inputs) if (inp.number() == unitig->number) return {};
    return inputs;
}

std::vector<UnitigStrand> get_exclusive_outputs(const Unitig* unitig) {   // :258-280
    std::vector<UnitigStrand> outputs;
    for (auto& next : unitig->forward_next) {
        auto& prevs = next.strand ? next.unitig->forward_prev : next.unitig->reverse_prev;
        bool exclusive = prevs.size() == 1 && prevs[0].strand && prevs[0].number() == unitig->number;
        if (!exclusive) return {};
        outputs.push_back(next);
    }
    for (auto& o : outputs) if (o.number() == unitig->number) return {};
    return outputs;
}

static bool starts_with(const std::string& s, const std::string& p) { return s.size() >= p.size() && s.compare(0, p.size(), p) == 0; }

std::string get_common_start_seq(const std::vector<UnitigStrand>& unitigs) {   // :283-295
    if (unitigs.empty()) return {};
    std::vector<std::string> seqs; for (auto& u : unitigs) seqs.push_back(u.unitig->get_seq(u.strand));
    std::string prefix = seqs[0];
    for (auto& seq : seqs)
        while (!starts_with(seq, prefix)) { prefix.pop_back(); if (prefix.empty()) return {}; }
    return prefix;
}

std::string get_common_end_seq(const std::vector<UnitigStrand>& unitigs) {   // :298-312
    if (unitigs.empty()) return {};
    std::vector<std::string> seqs;
    for (auto& u : unitigs) { std::string s = u.unitig->get_seq(u.strand); std::reverse(s.begin(), s.end()); seqs.push_back(s); }
    std::string suffix = seqs[0];
    for (auto& seq : seqs)
        while (!starts_with(seq, suffix)) { suffix.pop_back(); if (suffix.empty()) return {}; }
    std::reverse(suffix.begin(), suffix.end());
    return suffix;
}

static bool check_for_duplicates(const std::vector<UnitigStrand>& unitigs) {   // :184-187
    std::unordered_set<uint32_t> s; for (auto& u : unitigs) s.insert(u.number());
    return s.size() != unitigs.size();
}

static void avoid_zero_len_unitigs(std::string& common_seq, const std::vector<UnitigStrand>& sources, bool trim_from_start) {   // :141-158
    if (common_seq.empty()) return;
    uint32_t dup = check_for_duplicates(sources) ? 2 : 1;
    uint32_t min_source_len = UINT32_MAX;
    for (auto& s : sources) min_source_len = std::min(min_source_len, s.unitig->length());
    while (min_source_len <= (uint32_t)common_seq.size() * dup) {
        if (trim_from_start) common_seq.erase(0, 1); else common_seq.pop_back();
    }
}

static void avoid_start_of_path(std::string& common_seq, const Unitig* dest, bool trim_from_start) {   // :161-181
    if (common_seq.empty()) return;
    auto any_le = [&](const std::vector<Position>& ps) { for (auto& p : ps) if (p.pos <= (uint32_t)common_seq.size()) return true; return false; };
    if (trim_from_start) { while (any_le(dest->forward_positions)) common_seq.erase(0, 1); }
    else { while (any_le(dest->reverse_positions)) common_seq.pop_back(); }
}

static size_t shift_sequence_1(const std::vector<UnitigStrand>& sources, Unitig* dest) {   // :89-116
    std::string common_seq = get_common_end_seq(sources);
    avoid_zero_len_unitigs(common_seq, sources, true);
    avoid_start_of_path(common_seq, dest, true);
    size_t shifted = common_seq.size();
    if (shifted == 0) return 0;
    for (auto& s : sources) { if (s.strand) s.unitig->remove_seq_from_end(shifted); else s.unitig->remove_seq_from_start(shifted); }
    dest->add_seq_to_start(common_seq);
    return shifted;
}

static size_t shift_sequence_2(Unitig* dest, const std::vector<UnitigStrand>& sources) {   // :119-138
    std::string common_seq = get_common_start_seq(sources);
    avoid_zero_len_unitigs(common_seq, sources, false);
    avoid_start_of_path(common_seq, dest, false);
    size_t shifted = common_seq.size();
    if (shifted == 0) return 0;
    for (auto& s : sources) { if (s.strand) s.unitig->remove_seq_from_start(shifted); else s.unitig->remove_seq_from_end(shifted); }
    dest->add_seq_to_end(common_seq);
    return shifted;
}

static void get_fixed_unitig_starts_and_ends(const UnitigGraph& graph, const std::vector<Sequence>& sequences,
                                             std::unordered_set<uint32_t>& fixed_starts, std::unordered_set<uint32_t>& fixed_ends) {   // :190-230
    for (auto& seq : sequences) {
        auto path = graph.get_unitig_path_for_sequence(seq);
        if (path.empty()) continue;
        if (path.front().second) fixed_starts.insert(path.front().first); else fixed_ends.insert(path.front().first);
        if (path.back().second) fixed_ends.insert(path.back().first); else fixed_starts.insert(path.back().first);
    }
    auto starts_copy = fixed_starts; auto ends_copy = fixed_ends;
    for (uint32_t u : starts_copy)
        for (auto& up : graph.unitig_index.at(u)->forward_prev) { if (up.strand) fixed_ends.insert(up.number()); else fixed_starts.insert(up.number()); }
    for (uint32_t u : ends_copy)
        for (auto& down : graph.unitig_index.at(u)->forward_next) { if (down.strand) fixed_starts.insert(down.number()); else fixed_ends.insert(down.number()); }
}

size_t expand_repeats(UnitigGraph& graph, const std::vector<Sequence>& seqs) {   // :43-86
    std::unordered_set<uint32_t> fixed_starts, fixed_ends;
    get_fixed_unitig_starts_and_ends(graph, seqs, fixed_starts, fixed_ends);
    size_t total = 0;
    for (auto& up : graph.unitigs) {
        Unitig* u = up.get();
        uint32_t num = u->number;
        auto inputs = get_exclusive_inputs(u);
        if (inputs.size() >= 2 && !fixed_starts.count(num)) {
            bool can_shift = true;
            for (auto& in : inputs)
                if ((in.strand && fixed_ends.count(in.number())) || (!in.strand && fixed_starts.count(in.number()))) { can_shift = false; break; }
            if (can_shift) total += shift_sequence_1(inputs, u);
        }
        auto outputs = get_exclusive_outputs(u);
        if (outputs.size() >= 2 && !fixed_ends.count(num)) {
            bool can_shift = true;
            for (auto& o : outputs)
                if ((o.strand && fixed_starts.count(o.number())) || (!o.strand && fixed_ends.count(o.number()))) { can_shift = false; break; }
            if (can_shift) total += shift_sequence_2(u, outputs);
        }
    }
    return total;
}

void simplify_structure(UnitigGraph& graph, const std::vector<Sequence>& seqs) {   // :26-40
    while (expand_repeats(graph, seqs) > 0) {}
    graph.renumber_unitigs();
}

// ---------------------------------------------------------------------------------------------
// graph_simplification.rs:315-526 merge_linear_paths and the UnitigGraph helpers it uses
// ---------------------------------------------------------------------------------------------
void UnitigGraph::delete_dangling_links() {   // unitig_graph.rs:547-564: links are kept or dropped by unitig NUMBER
    std::unordered_set<uint32_t> numbers;
    for (auto& u : unitigs) numbers.insert(u->number);
    auto prune = [&](std::vector<UnitigStrand>& v) {
        std::vector<UnitigStrand> kept;
        for (auto& l : v) if (numbers.count(l.number())) kept.push_back(l);
        v.swap(kept);
    };
    for (auto& u : unitigs) { prune(u->forward_next); prune(u->forward_prev); prune(u->reverse_next); prune(u->reverse_prev); }
}

uint32_t UnitigGraph::max_unitig_number() const {   // unitig_graph.rs:901-903
    uint32_t m = 0; for (auto& u : unitigs) m = std::max(m, u->number); return m;
}

std::vector<std::vector<uint32_t>> UnitigGraph::connected_components() const {   // unitig_graph.rs:905-947
    std::unordered_set<uint32_t> visited;
    std::vector<std::vector<uint32_t>> components;
    for (auto& u : unitigs) {
        if (visited.count(u->number)) continue;
        std::vector<uint32_t> component, stack{u->number};
        while (!stack.empty()) {
            const uint32_t cur = stack.back(); stack.pop_back();
            if (!visited.insert(cur).second) continue;
            component.push_back(cur);
            auto it = unitig_index.find(cur);
            if (it == unitig_index.end()) continue;
            const Unitig* c = it->second;
            for (auto* v : {&c->forward_next, &c->forward_prev, &c->reverse_next, &c->reverse_prev})
                for (auto& l : *v) if (!visited.count(l.number())) stack.push_back(l.number());
        }
        std::sort(component.begin(), component.end());
        components.push_back(std::move(component));
    }
    std::sort(components.begin(), components.end());
    return components;
}

bool UnitigGraph::component_is_circular_loop(const std::vector<uint32_t>& component) const {   // unitig_graph.rs:949-967
    if (component.empty()) return false;
    const uint32_t first = component[0];
    uint32_t num = first; bool strand = strand::FORWARD;
    std::unordered_set<uint32_t> visited;
    while (num != first || visited.empty()) {
        if (!visited.insert(num).second) return false;
        const Unitig* u = unitig_index.at(num);
        if (u->forward_next.size() != 1 || u->forward_prev.size() != 1 || u->reverse_next.size() != 1 || u->reverse_prev.size() != 1) return false;
        const UnitigStrand& next = strand ? u->forward_next[0] : u->reverse_next[0];
        num = next.number(); strand = next.strand;
    }
    return visited.size() == component.size();
}

void merge_fixed_sets(const UnitigGraph& graph, const std::vector<Sequence>& seqs, std::unordered_set<uint32_t>& fixed_starts,
                      std::unordered_set<uint32_t>& fixed_ends) {   // :330-331, fix_circular_loops :374-384
    get_fixed_unitig_starts_and_ends(graph, seqs, fixed_starts, fixed_ends);
    for (auto& component : graph.connected_components())
        if (graph.component_is_circular_loop(component)) fixed_starts.insert(component[0]);
}

static bool cannot_merge_start(uint32_t n, bool s, const std::unordered_set<uint32_t>& fs, const std::unordered_set<uint32_t>& fe) {   // :387-390
    return (s && fs.count(n)) || (!s && fe.count(n));
}
static bool cannot_merge_end(uint32_t n, bool s, const std::unordered_set<uint32_t>& fs, const std::unordered_set<uint32_t>& fe) {     // :398-401
    return (s && fe.count(n)) || (!s && fs.count(n));
}

std::string merge_unitig_seqs(const std::vector<UnitigStrand>& path) {   // :490-500
    std::string merged;
    for (auto& u : path) merged += u.unitig->get_seq(u.strand);
    return merged;
}

static double get_merge_path_depth(const std::vector<UnitigStrand>& path, const std::vector<Position>& forward_positions) {   // :503-526
    if (!forward_positions.empty()) return (double)forward_positions.size();
    for (auto& u : path) if (u.unitig->unitig_type == UnitigType::Anchor) return u.unitig->depth;
    double total = 0.0, sum = 0.0;
    { uint32_t t = 0; for (auto& u : path) t += u.unitig->length(); total = (double)t; }
    for (auto& u : path) sum += u.unitig->depth * (double)u.unitig->length();
    return sum / total;
}

static void merge_path(UnitigGraph& graph, const std::vector<UnitigStrand>& path, uint32_t new_number) {   // :410-487
    const UnitigStrand first = path.front(), last = path.back();
    auto nu = std::make_unique<Unitig>();
    Unitig* n = nu.get();
    n->number = new_number;
    n->forward_seq = merge_unitig_seqs(path);
    n->reverse_seq = reverse_complement(n->forward_seq);
    n->forward_positions = first.strand ? first.unitig->forward_positions : first.unitig->reverse_positions;
    n->reverse_positions = last.strand ? last.unitig->reverse_positions : last.unitig->forward_positions;
    const bool end_to_start = graph.link_exists(last.number(), last.strand, first.number(), first.strand);
    const bool start_flip = graph.link_exists(first.number(), !first.strand, first.number(), first.strand);
    const bool end_flip = graph.link_exists(last.number(), last.strand, last.number(), !last.strand);
    n->forward_prev = first.strand ? first.unitig->forward_prev : first.unitig->reverse_prev;
    n->reverse_next = first.strand ? first.unitig->reverse_next : first.unitig->forward_next;
    n->forward_next = last.strand ? last.unitig->forward_next : last.unitig->reverse_next;
    n->reverse_prev = last.strand ? last.unitig->reverse_prev : last.unitig->forward_prev;
    n->depth = get_merge_path_depth(path, n->forward_positions);
    for (auto& p : path)
        if (p.unitig->unitig_type == UnitigType::Anchor || p.unitig->unitig_type == UnitigType::Consentig) n->unitig_type = UnitigType::Consentig;
    graph.unitigs.push_back(std::move(nu));

    // links from the neighbours to the new unitig (:446-461); copies, because a neighbour may be the new unitig's own list owner
    const auto f_next = n->forward_next, f_prev = n->forward_prev, r_next = n->reverse_next, r_prev = n->reverse_prev;
    for (auto& u : f_next) (u.strand ? u.unitig->forward_prev : u.unitig->reverse_prev).push_back(UnitigStrand{n, strand::FORWARD});
    for (auto& u : f_prev) (u.strand ? u.unitig->forward_next : u.unitig->reverse_next).push_back(UnitigStrand{n, strand::FORWARD});
    for (auto& u : r_next) (u.strand ? u.unitig->forward_prev : u.unitig->reverse_prev).push_back(UnitigStrand{n, strand::REVERSE});
    for (auto& u : r_prev) (u.strand ? u.unitig->forward_next : u.unitig->reverse_next).push_back(UnitigStrand{n, strand::REVERSE});

    if (end_to_start) {   // :464-470
        n->forward_next.push_back(UnitigStrand{n, strand::FORWARD}); n->forward_prev.push_back(UnitigStrand{n, strand::FORWARD});
        n->reverse_next.push_back(UnitigStrand{n, strand::REVERSE}); n->reverse_prev.push_back(UnitigStrand{n, strand::REVERSE});
    }
    if (start_flip) { n->reverse_next.push_back(UnitigStrand{n, strand::FORWARD}); n->forward_prev.push_back(UnitigStrand{n, strand::REVERSE}); }
    if (end_flip) { n->forward_next.push_back(UnitigStrand{n, strand::REVERSE}); n->reverse_prev.push_back(UnitigStrand{n, strand::FORWARD}); }

    std::unordered_set<uint32_t> path_numbers;   // :485-486
    for (auto& p : path) path_numbers.insert(p.number());
    std::vector<std::unique_ptr<Unitig>> kept;
    for (auto& u : graph.unitigs) { if (path_numbers.count(u->number)) graph.retired.push_back(std::move(u)); else kept.push_back(std::move(u)); }
    graph.unitigs.swap(kept);
}

void merge_linear_paths(UnitigGraph& graph, const std::vector<Sequence>& seqs) {   // :315-371
    std::unordered_set<uint32_t> fixed_starts, fixed_ends;
    merge_fixed_sets(graph, seqs, fixed_starts, fixed_ends);
    std::unordered_set<uint32_t> already_used;
    std::vector<std::vector<UnitigStrand>> merge_paths;
    for (auto& up : graph.unitigs) {
        Unitig* unitig = up.get();
        for (bool unitig_strand : {strand::FORWARD, strand::REVERSE}) {
            if (already_used.count(unitig->number)) continue;
            const auto inputs = unitig_strand ? get_exclusive_inputs(unitig) : get_exclusive_outputs(unitig);
            if (inputs.size() == 1 && !cannot_merge_start(unitig->number, unitig_strand, fixed_starts, fixed_ends)) continue;
            std::vector<UnitigStrand> current{UnitigStrand{unitig, unitig_strand}};
            already_used.insert(unitig->number);
            for (;;) {
                const UnitigStrand u = current.back();
                if (cannot_merge_end(u.number(), u.strand, fixed_starts, fixed_ends)) break;
                auto outputs = u.strand ? get_exclusive_outputs(u.unitig) : get_exclusive_inputs(u.unitig);
                if (outputs.size() != 1) break;
                UnitigStrand output = outputs[0];
                if (!u.strand) output.strand = !output.strand;
                if (already_used.count(output.number())) break;
                if (cannot_merge_start(output.number(), output.strand, fixed_starts, fixed_ends)) break;
                current.push_back(output);
                already_used.insert(output.number());
            }
            if (current.size() > 1) merge_paths.push_back(current);
        }
    }
    uint32_t new_number = graph.max_unitig_number();
    for (auto& path : merge_paths) merge_path(graph, path, ++new_number);
    graph.delete_dangling_links();
    graph.build_unitig_index();
    graph.check_links();
}

// ---------------------------------------------------------------------------------------------
// cluster.rs:132-176 pairwise_contig_distances + save_distance_matrix
// ---------------------------------------------------------------------------------------------
std::string pairwise_distance_matrix(const UnitigGraph& graph, const std::vector<Sequence>& sequences) {
    std::unordered_map<uint32_t, uint32_t> unitig_lengths;
    for (auto& u : graph.unitigs) unitig_lengths[u->number] = u->length();
    std::unordered_map<uint16_t, std::unordered_set<uint32_t>> sequence_unitigs;
    for (auto& s : sequences) {
        std::unordered_set<uint32_t> set;
        for (auto& step : graph.get_unitig_path_for_sequence(s)) set.insert(step.first);
        sequence_unitigs[s.id] = std::move(set);
    }
    std::map<std::pair<uint16_t, uint16_t>, double> distances;
    for (auto& seq_a : sequences) {
        const auto& a = sequence_unitigs.at(seq_a.id);
        uint32_t a_sum = 0; for (uint32_t u : a) a_sum += unitig_lengths.at(u);      // sum::<u32>()
        const double a_len = (double)a_sum;
        for (auto& seq_b : sequences) {
            const auto& b = sequence_unitigs.at(seq_b.id);
            double ab_len = 0.0;                                                       // f64 sum of whole numbers: exact in any order
            for (uint32_t u : a) if (b.count(u)) ab_len += (double)unitig_lengths.at(u);
            distances[{seq_a.id, seq_b.id}] = 1.0 - (ab_len / a_len);
        }
    }
    std::string out = std::to_string(sequences.size()) + "\n";
    for (auto& seq_a : sequences) {
        out += seq_a.display();
        for (auto& seq_b : sequences) { char buf[64]; snprintf(buf, sizeof buf, "\t%.8f", distances.at({seq_a.id, seq_b.id})); out += buf; }
        out += "\n";
    }
    return out;
}

// ---------------------------------------------------------------------------------------------
// decompress.rs:83-114
// ---------------------------------------------------------------------------------------------
void save_original_seqs_to_dir(const std::string& out_dir, const UnitigGraph& g, const std::vector<Sequence>& seqs) {
    std::map<std::string, std::vector<std::pair<std::string, std::string>>> original;   // filenames.sort() => ordered map
    for (auto& s : seqs) original[s.filename].emplace_back(s.contig_header, g.reconstruct_original_sequence(s));
    for (auto& kv : original) {
        std::string path = out_dir + "/" + kv.first, text;
        for (auto& hs : kv.second) text += ">" + hs.first + "\n" + hs.second + "\n";
        std::string stem, ext; split_ext(kv.first, stem, ext);
        if (ext == "gz") {
            gzFile f = gzopen(path.c_str(), "wb"); if (!f) quit_with_error("cannot write " + path);
            gzwrite(f, text.data(), (unsigned)text.size()); gzclose(f);
        } else {
            std::ofstream f(path, std::ios::binary); f << text;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// metrics.rs:65-107,250-254 — serde_yaml 0.9 rendering of InputAssemblyMetrics
// ---------------------------------------------------------------------------------------------
static bool yaml_plain_ok(const std::string& s) {
    if (s.empty()) return false;
    static const char* ambiguous[] = {"~", "null", "Null", "NULL", "true", "True", "TRUE", "false", "False", "FALSE",
                                      "y", "Y", "yes", "Yes", "YES", "n", "N", "no", "No", "NO", "on", "On", "ON", "off", "Off", "OFF",
                                      ".nan", ".NaN", ".NAN", ".inf", ".Inf", ".INF", "-.inf", "-.Inf", "-.INF", "+.inf", "+.Inf", "+.INF"};
    for (auto a : ambiguous) if (s == a) return false;
    { char* e = nullptr; strtod(s.c_str(), &e); if (e && *e == 0) return false; }   // looks numeric
    if (s.front() == ' ' || s.back() == ' ') return false;
    if (strchr("-?:,[]{}#&*!|>'\"%@`", s.front())) {
        if (!((s.front() == '-' || s.front() == '?' || s.front() == ':') && s.size() > 1 && s[1] != ' ')) return false;
    }
    for (size_t i = 0; i < s.size(); ++i) {
        unsigned char c = s[i];
        if (c < 0x20 || c == 0x7f) return false;
        if (c == ':' && (i + 1 == s.size() || s[i + 1] == ' ')) return false;
        if (c == '#' && i > 0 && s[i - 1] == ' ') return false;
    }
    return true;
}
static std::string yaml_str(const std::string& s) {
    if (yaml_plain_ok(s)) return s;
    std::string q = "'"; for (char c : s) { q += c; if (c == '\'') q += '\''; } q += "'"; return q;
}
std::string InputAssemblyMetrics::to_yaml() const {
    std::string y;
    y += "input_assemblies_count: " + std::to_string(input_assemblies_count) + "\n";
    y += "input_assemblies_total_contigs: " + std::to_string(input_assemblies_total_contigs) + "\n";
    y += "input_assemblies_total_length: " + std::to_string(input_assemblies_total_length) + "\n";
    y += "compressed_unitig_count: " + std::to_string(compressed_unitig_count) + "\n";
    y += "compressed_unitig_total_length: " + std::to_string(compressed_unitig_total_length) + "\n";
    if (input_assembly_details.empty()) { y += "input_assembly_details: []\n"; return y; }
    y += "input_assembly_details:\n";
    for (auto& a : input_assembly_details) {
        y += "- filename: " + yaml_str(a.filename) + "\n";
        if (a.contigs.empty()) { y += "  contigs: []\n"; continue; }
        y += "  contigs:\n";
        for (auto& c : a.contigs) {
            y += "  - name: " + yaml_str(c.name) + "\n";
            y += "    description: " + yaml_str(c.description) + "\n";
            y += "    length: " + std::to_string(c.length) + "\n";
        }
    }
    return y;
}

}  // namespace orc
