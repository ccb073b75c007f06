// `autocycler clean`, `autocycler gfa2fasta` and `autocycler table` (host_clean.h).  The graph edits restate unitig_graph.rs:547-721
// literally on per-strand link lists (EditGraph), including the order of every list entry: the L-line order of the output depends on it.
#include "host_clean.h"

#include <dirent.h>
#include <sys/stat.h>

#include <algorithm>
#include <cctype>
#include <charconv>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>
#include <stdexcept>

#include "host_edit.h"
#include "host_io.h"

// ------------------------------------------------------------------------------------------------
// the graph edits (unitig_graph.rs:588-721) and the isolated-unitig tests (unitig.rs:275-292)
// ------------------------------------------------------------------------------------------------
void HostGraph::remove_unitigs(const std::vector<uint32_t>& numbers) {
    EditGraph e;
    e.from(*this);
    const std::set<uint32_t> gone(numbers.begin(), numbers.end());
    std::vector<uint8_t> keep(e.number.size());
    for (size_t u = 0; u < keep.size(); ++u) keep[u] = !gone.count(e.number[u]);
    e.retain(keep);
    e.to(*this);
    set_position_counts(e.visits);
}

void HostGraph::duplicate_unitig(uint32_t num) {
    EditGraph e;
    e.from(*this);
    const auto it = e.index.find(num);
    if (it == e.index.end()) throw InputError{"unitig " + std::to_string(num) + " not found in unitig index"};
    const uint32_t t = it->second;
    auto signed_of = [&](UStrand s) { const int32_t n = (int32_t)e.number[us_index(s)]; return us_reverse(s) ? -n : n; };
    // check_if_unitig_can_be_duplicated (:657-668), and the links the copies take over, from forward_next then reverse_next
    std::vector<std::pair<int32_t, int32_t>> non_self;
    std::vector<std::pair<bool, bool>> self_links;       // (from the reverse strand, to the reverse strand)
    for (uint32_t r = 0; r < 2; ++r)
        for (UStrand s : e.nx[2 * (size_t)t + r]) {
            if (e.number[us_index(s)] != num) non_self.emplace_back(r ? -(int32_t)num : (int32_t)num, signed_of(s));
            else self_links.emplace_back(r != 0, us_reverse(s));
        }
    if (non_self.size() != 2) throw InputError{"unitig " + std::to_string(num) + " does not contain exactly two non-self links"};
    const uint32_t a = *std::max_element(e.number.begin(), e.number.end()) + 1, b = a + 1;   // max_unitig_number before the removal
    const std::string seq = e.seq[t];
    const double depth = e.depth[t] / 2.0;
    const uint8_t type = e.type[t];
    const uint32_t visits = e.visits[t];                 // the copies are clones: they keep the positions
    e.visits[e.add_unitig(a, std::string(seq), depth, type)] = visits;
    e.visits[e.add_unitig(b, std::string(seq), depth, type)] = visits;
    std::vector<uint8_t> keep(e.number.size());
    for (size_t u = 0; u < keep.size(); ++u) keep[u] = e.number[u] != num;
    e.retain(keep);
    const int32_t sa = (int32_t)a, sb = (int32_t)b;
    for (const auto& l : self_links) {                   // loops and hairpins, each link once per copy (create_link adds the mirror)
        e.create_link(e.strand(l.first ? -sa : sa), e.strand(l.second ? -sa : sa));
        e.create_link(e.strand(l.first ? -sb : sb), e.strand(l.second ? -sb : sb));
    }
    auto replace = [&](int32_t x, int32_t with) { return (x < 0 ? -x : x) == (int32_t)num ? (x < 0 ? -with : with) : x; };   // find_replace_i32_tuple (misc.rs:509-515)
    e.create_link(e.strand(replace(non_self[0].first, sa)), e.strand(replace(non_self[0].second, sa)));
    e.create_link(e.strand(replace(non_self[1].first, sb)), e.strand(replace(non_self[1].second, sb)));
    e.to(*this);                                          // ends with check_links
    set_position_counts(e.visits);
}

void HostGraph::remove_low_depth_unitigs(double min_depth) {
    EditGraph e;
    e.from(*this);
    const size_t n0 = e.number.size();
    for (size_t idx = n0; idx-- > 0;) {                   // in reverse, to keep longer unitigs
        if (idx >= e.number.size()) continue;
        const uint32_t num = e.number[idx];
        if (e.depth[idx] > min_depth) continue;
        // every neighbour must keep a link on the side it shares with this unitig: a next strand on its prev list, a prev strand on
        // its next list
        auto keeps_other = [&](const std::vector<UStrand>& list) {
            for (UStrand l : list) if (e.number[us_index(l)] != num) return true;
            return false;
        };
        bool ok = true;
        for (UStrand s : e.nx[2 * idx]) if (e.number[us_index(s)] != num && !keeps_other(e.pv[s])) { ok = false; break; }
        if (ok) for (UStrand s : e.pv[2 * idx]) if (e.number[us_index(s)] != num && !keeps_other(e.nx[s])) { ok = false; break; }
        if (!ok) continue;
        std::vector<uint8_t> keep(e.number.size());
        for (size_t u = 0; u < keep.size(); ++u) keep[u] = e.number[u] != num;
        e.retain(keep);
    }
    e.to(*this);
    set_position_counts(e.visits);
}

void HostGraph::set_position_counts(const std::vector<uint32_t>& counts) {
    own_path.clear();
    for (uint32_t u = 0; u < U; ++u) own_path.insert(own_path.end(), counts[u], us_make(u, false));
    own_path_off.assign({0, (uint64_t)own_path.size()});
    path_off = own_path_off.data(); path = own_path.data(); n_path = own_path.size(); n_seqs = 1;
}

bool HostGraph::is_isolated_and_circular(uint32_t idx) const {
    const UStrand fw = us_make(idx, false);
    return next_size(fw) == 1 && prev_size(fw) == 1 && next_begin(fw)[0] == fw && prev_begin(fw)[0] == fw;
}

bool HostGraph::is_isolated_and_linear(uint32_t idx) const {
    const UStrand fw = us_make(idx, false), rv = us_make(idx, true);
    if (next_size(fw) > 1 || prev_size(fw) > 1 || is_isolated_and_circular(idx)) return false;
    auto all_are = [](const UStrand* b, uint32_t n, UStrand x) { for (uint32_t i = 0; i < n; ++i) if (b[i] != x) return false; return true; };
    return all_are(next_begin(fw), next_size(fw), rv) && all_are(prev_begin(fw), prev_size(fw), rv) &&
           all_are(next_begin(rv), next_size(rv), fw) && all_are(prev_begin(rv), prev_size(rv), fw);
}

// ------------------------------------------------------------------------------------------------
// clean (clean.rs:23-149)
// ------------------------------------------------------------------------------------------------
namespace {
void graph_info(bool verbose, const HostGraph& g) {     // print_basic_graph_info (unitig_graph.rs:509-516)
    if (verbose) fprintf(stderr, "%u unitig%s, %llu link%s\ntotal length: %llu bp\n\n", g.U, g.U == 1 ? "" : "s", (unsigned long long)g.link_count_single(),
                         g.link_count_single() == 1 ? "" : "s", (unsigned long long)g.total_length());
}
void section(bool verbose, const char* title, const char* explanation) {
    if (verbose) fprintf(stderr, "\n%s\n    %s\n\n", title, explanation);
}
}  // namespace

std::vector<uint32_t> parse_tig_numbers(const std::string& text) {
    std::string t;
    for (char c : text) if (c != ' ') t += c;
    std::vector<uint32_t> out;
    size_t a = 0;
    while (true) {
        const size_t b = std::min(t.find(',', a), t.size());
        const std::string item = t.substr(a, b - a);
        // str::parse::<u32>: an optional '+', then digits only, no overflow
        size_t i = !item.empty() && item[0] == '+' ? 1 : 0;
        uint64_t v = 0;
        bool good = i < item.size();
        for (; good && i < item.size(); ++i) {
            if (item[i] < '0' || item[i] > '9') good = false;
            else if ((v = v * 10 + (uint64_t)(item[i] - '0')) > 0xFFFFFFFFull) good = false;
        }
        if (!good) throw InputError{"failed to parse '" + item + "' as a node number"};
        out.push_back((uint32_t)v);
        if (b == t.size()) break;
        a = b + 1;
    }
    std::sort(out.begin(), out.end());
    return out;
}

void load_user_gfa(const std::string& text, HostGraph& g) {
    std::vector<HostSeq> seqs;
    try { g.load_gfa(text.data(), text.size(), seqs); }
    catch (const std::runtime_error& e) { throw InputError{e.what()}; }
}

void clean_graph(HostGraph& g, const std::string& name, std::vector<uint32_t> remove, std::vector<uint32_t> duplicate,
                 const double* min_depth, bool merge, bool verbose, std::string& gfa) {
    std::sort(remove.begin(), remove.end());
    std::sort(duplicate.begin(), duplicate.end());
    std::set<uint32_t> all;                               // check_tig_numbers_are_valid (:128-139): --remove, then --duplicate
    for (uint32_t u = 0; u < g.U; ++u) all.insert(g.number[u]);
    for (const std::vector<uint32_t>* list : {&remove, &duplicate})
        for (uint32_t n : *list) if (!all.count(n)) throw InputError{name + " does not contain tig " + std::to_string(n)};
    for (uint32_t n : duplicate) if (std::binary_search(remove.begin(), remove.end(), n))
        throw InputError{"tig " + std::to_string(n) + " cannot be both removed and duplicated"};
    for (size_t i = 1; i < duplicate.size(); ++i) if (duplicate[i] == duplicate[i - 1])
        throw InputError{"tig " + std::to_string(duplicate[i]) + " cannot be duplicated more than once"};
    if (!remove.empty()) {
        section(verbose, "Removing sequences", "The user-specified tigs are now removed from the graph.");
        g.remove_unitigs(remove);
        graph_info(verbose, g);
    }
    if (!duplicate.empty()) {
        section(verbose, "Duplicating sequences", "The user-specified tigs are now duplicated in the graph.");
        for (uint32_t n : duplicate) g.duplicate_unitig(n);
        graph_info(verbose, g);
    }
    if (min_depth) {
        section(verbose, "Removing low depth sequences", "Tigs with a depth below the specified threshold are now removed from the graph, "
                                                         "if and only if doing so would not create a dead end.");
        g.remove_low_depth_unitigs(*min_depth);
        graph_info(verbose, g);
    }
    if (merge) {
        section(verbose, "Merging linear paths", "Linear paths in the graph are now merged.");
        g.merge_linear_paths(false);
        graph_info(verbose, g);
        g.renumber();
    }
    const std::vector<HostSeq> none;
    g.gfa_text(none, gfa, true);
}

// ------------------------------------------------------------------------------------------------
// gfa2fasta (gfa2fasta.rs:55-82)
// ------------------------------------------------------------------------------------------------
std::string gfa_fasta_text(const HostGraph& g, uint64_t counts[3]) {
    std::string out;
    counts[0] = counts[1] = counts[2] = 0;
    for (uint32_t n = 0; n < g.U; ++n) {                  // the loaded order: the file's S lines
        const uint32_t u = g.order[n];
        if (g.rec[u].len == 0) continue;
        const char* topology = "";
        if (g.is_isolated_and_circular(u)) { topology = " circular=true topology=circular"; counts[0] += 1; }
        else if (g.is_isolated_and_linear(u)) { topology = " circular=false topology=linear"; counts[1] += 1; }
        else counts[2] += 1;
        out += ">" + std::to_string(g.number[u]) + " length=" + std::to_string(g.rec[u].len) + topology + "\n";
        out.append(g.seq_ptr(u), g.rec[u].len);
        out += "\n";
    }
    return out;
}

// ------------------------------------------------------------------------------------------------
// table (table.rs:24-204) and what it reads
// ------------------------------------------------------------------------------------------------
const char* const TABLE_DEFAULT_FIELDS =
    "input_read_count, input_read_bases, input_read_n50, pass_cluster_count, fail_cluster_count, overall_clustering_score, "
    "untrimmed_cluster_size, untrimmed_cluster_distance, trimmed_cluster_size, trimmed_cluster_median, trimmed_cluster_mad, "
    "consensus_assembly_bases, consensus_assembly_unitigs, consensus_assembly_fully_resolved";

namespace {
// get_field_names of SubsampleMetrics, InputAssemblyMetrics, ClusteringMetrics, UntrimmedClusterMetrics, TrimmedClusterMetrics and
// CombineMetrics (metrics.rs:333-358)
const char* const FIELD_NAMES[] = {
    "input_read_bases", "input_read_count", "input_read_n50", "output_reads",
    "compressed_unitig_count", "compressed_unitig_total_length", "input_assemblies_count", "input_assemblies_total_contigs",
    "input_assemblies_total_length", "input_assembly_details",
    "cluster_balance_score", "cluster_tightness_score", "fail_cluster_count", "fail_contig_count", "fail_contig_fraction",
    "overall_clustering_score", "pass_cluster_count", "pass_contig_count", "pass_contig_fraction",
    "untrimmed_cluster_distance", "untrimmed_cluster_lengths", "untrimmed_cluster_mad", "untrimmed_cluster_median", "untrimmed_cluster_size",
    "trimmed_cluster_lengths", "trimmed_cluster_mad", "trimmed_cluster_median", "trimmed_cluster_size",
    "consensus_assembly_bases", "consensus_assembly_clusters", "consensus_assembly_fully_resolved", "consensus_assembly_unitigs"};

// serde_yaml::Value, as much of it as table formats
struct YValue {
    enum Kind { Null, Bool, Int, Float, Str, Seq, Map } kind = Null;
    bool b = false;
    std::string text;                                     // Int: the decimal digits; Str: the string
    double f = 0;
    std::vector<YValue> items;                            // Seq: the items; Map: key, value, key, value, ...
};

struct YamlError {};

// __powidf2 (compiler-rt), which 10f64.powi(d) calls: square-and-multiply, and 1 / r for a negative exponent
double powi(double a, int32_t b) {
    const bool recip = b < 0;
    double r = 1;
    while (true) {
        if (b & 1) r *= a;
        b /= 2;
        if (b == 0) break;
        a *= a;
    }
    return recip ? 1 / r : r;
}

int32_t saturating_i32(double x) {                        // `as i32`: NaN is 0, out-of-range values saturate
    if (std::isnan(x)) return 0;
    if (x >= 2147483647.0) return 2147483647;
    if (x <= -2147483648.0) return INT32_MIN;
    return (int32_t)x;
}

std::string fixed(double v, int64_t decimals) {          // format!("{:.N}") for finite and non-finite values
    if (std::isnan(v)) return "NaN";
    if (std::isinf(v)) return v < 0 ? "-inf" : "inf";
    const int n = snprintf(nullptr, 0, "%.*f", (int)decimals, v);
    std::string s((size_t)n + 1, '\0');
    snprintf(&s[0], s.size(), "%.*f", (int)decimals, v);
    s.resize((size_t)n);
    return s;
}

std::string shortest(double v) {                          // format!("{}"): the shortest round-trip digits in fixed notation, zero-padded
    if (std::isnan(v)) return "NaN";
    if (std::isinf(v)) return v < 0 ? "-inf" : "inf";
    // to_chars' fixed form would print a large integer's exact digits; Rust pads the shortest digits with zeros instead
    char buf[64];
    const auto r = std::to_chars(buf, buf + sizeof buf, v, std::chars_format::scientific);
    const std::string sci(buf, r.ptr);
    const size_t e = sci.find('e');
    const int exp10 = atoi(sci.c_str() + e + 1);
    std::string digits, out = sci[0] == '-' ? "-" : "";
    for (size_t i = sci[0] == '-' ? 1 : 0; i < e; ++i) if (sci[i] != '.') digits += sci[i];
    const int point = exp10 + 1;                         // digits before the decimal point
    if (point <= 0) return out + "0." + std::string((size_t)-point, '0') + digits;
    if ((size_t)point >= digits.size()) return out + digits + std::string((size_t)point - digits.size(), '0');
    return out + digits.substr(0, (size_t)point) + "." + digits.substr((size_t)point);
}
}  // namespace

std::string format_float_sigfigs(double value, uint64_t sigfigs) {
    const int32_t sf = (int32_t)(uint32_t)sigfigs;        // `sigfigs as i32`
    if (value == 0.0) return fixed(0.0, (int64_t)sigfigs - 1);
    const int32_t decimals = (int32_t)((uint32_t)sf - (uint32_t)saturating_i32(std::floor(std::log10(std::fabs(value)))) - 1u);   // wrapping, as a release build
    const double factor = powi(10.0, decimals);
    const double rounded = std::round(value * factor) / factor;
    return decimals > 0 ? fixed(rounded, decimals) : shortest(rounded);
}

namespace {
// ---- a reader for the YAML that serde_yaml 0.9 writes (and that this project's writers emit) ----
struct YLine { size_t indent; std::string text; };

bool digits_but_not_number(const std::string& s) {        // YAML 1.2: a leading zero followed by digits is a string
    const std::string t = !s.empty() && (s[0] == '-' || s[0] == '+') ? s.substr(1) : s;
    if (t.size() < 2 || t[0] != '0') return false;
    for (size_t i = 1; i < t.size(); ++i) if (t[i] < '0' || t[i] > '9') return false;
    return true;
}

bool parse_int(const std::string& s, YValue& v) {          // parse_unsigned_int / parse_negative_int: decimal, 0x, 0o, 0b
    if (s.empty() || digits_but_not_number(s)) return false;
    const bool neg = s[0] == '-';
    std::string t = s[0] == '+' || s[0] == '-' ? s.substr(1) : s;
    if (t.empty() || t[0] == '+' || t[0] == '-') return false;
    int base = 10;
    if (t.size() > 2 && t[0] == '0' && (t[1] == 'x' || t[1] == 'o' || t[1] == 'b')) { base = t[1] == 'x' ? 16 : t[1] == 'o' ? 8 : 2; t = t.substr(2); }
    unsigned __int128 x = 0;
    for (char c : t) {
        int d = c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : 99;
        if (d >= base) return false;
        x = x * (unsigned)base + (unsigned)d;
        if (x > ((unsigned __int128)1 << 64)) return false;
    }
    if (!neg && x > 0xFFFFFFFFFFFFFFFFull) return false;
    if (neg && x > ((unsigned __int128)1 << 63)) return false;
    v.kind = YValue::Int;
    if (neg && x != 0) { char buf[32]; snprintf(buf, sizeof buf, "-%llu", (unsigned long long)x); v.text = buf; }
    else v.text = std::to_string((unsigned long long)x);
    return true;
}

bool parse_float(const std::string& s, YValue& v) {        // parse_f64: .inf / .nan forms, else Rust's f64 grammar, finite results only
    std::string t = s;
    if (!t.empty() && t[0] == '+') { t = t.substr(1); if (!t.empty() && (t[0] == '+' || t[0] == '-')) return false; }
    v.kind = YValue::Float;
    if (t == ".inf" || t == ".Inf" || t == ".INF") { v.f = INFINITY; return true; }
    if (s == "-.inf" || s == "-.Inf" || s == "-.INF") { v.f = -INFINITY; return true; }
    if (s == ".nan" || s == ".NaN" || s == ".NAN") { v.f = NAN; return true; }
    size_t i = t.size() > 0 && t[0] == '-' ? 1 : 0, digits = 0;
    while (i < t.size() && isdigit((unsigned char)t[i])) { ++i; ++digits; }
    if (i < t.size() && t[i] == '.') { ++i; while (i < t.size() && isdigit((unsigned char)t[i])) { ++i; ++digits; } }
    if (digits == 0) return false;
    if (i < t.size() && (t[i] == 'e' || t[i] == 'E')) {
        ++i;
        if (i < t.size() && (t[i] == '+' || t[i] == '-')) ++i;
        size_t e = 0;
        while (i < t.size() && isdigit((unsigned char)t[i])) { ++i; ++e; }
        if (e == 0) return false;
    }
    if (i != t.size()) return false;
    v.f = strtod(t.c_str(), nullptr);
    return std::isfinite(v.f);
}

YValue plain_scalar(const std::string& s) {               // visit_untagged_scalar: null, bool, integer, float, else string
    YValue v;
    if (s.empty() || s == "~" || s == "null" || s == "Null" || s == "NULL") return v;
    if (s == "true" || s == "True" || s == "TRUE" || s == "false" || s == "False" || s == "FALSE") { v.kind = YValue::Bool; v.b = s[0] == 't' || s[0] == 'T'; return v; }
    if (parse_int(s, v)) return v;
    if (!digits_but_not_number(s) && parse_float(s, v)) return v;
    v = YValue(); v.kind = YValue::Str; v.text = s;
    return v;
}

void put_utf8(std::string& out, uint32_t c) {
    if (c < 0x80) out += (char)c;
    else if (c < 0x800) { out += (char)(0xC0 | (c >> 6)); out += (char)(0x80 | (c & 0x3F)); }
    else if (c < 0x10000) { out += (char)(0xE0 | (c >> 12)); out += (char)(0x80 | ((c >> 6) & 0x3F)); out += (char)(0x80 | (c & 0x3F)); }
    else { out += (char)(0xF0 | (c >> 18)); out += (char)(0x80 | ((c >> 12) & 0x3F)); out += (char)(0x80 | ((c >> 6) & 0x3F)); out += (char)(0x80 | (c & 0x3F)); }
}

// A quoted scalar starting at s[i]; i ends past the closing quote
std::string quoted(const std::string& s, size_t& i) {
    const char q = s[i++];
    std::string out;
    while (true) {
        if (i >= s.size()) throw YamlError{};
        const char c = s[i++];
        if (c == q) {
            if (q == '\'' && i < s.size() && s[i] == '\'') { out += '\''; ++i; continue; }
            return out;
        }
        if (q == '"' && c == '\\') {
            if (i >= s.size()) throw YamlError{};
            const char e = s[i++];
            switch (e) {
                case '0': out += '\0'; break;  case 'a': out += '\a'; break; case 'b': out += '\b'; break;
                case 't': case '\t': out += '\t'; break; case 'n': out += '\n'; break; case 'v': out += '\v'; break;
                case 'f': out += '\f'; break;  case 'r': out += '\r'; break; case 'e': out += '\x1b'; break;
                case ' ': out += ' '; break;   case '"': out += '"'; break;  case '/': out += '/'; break; case '\\': out += '\\'; break;
                case 'N': put_utf8(out, 0x85); break; case '_': put_utf8(out, 0xA0); break;
                case 'L': put_utf8(out, 0x2028); break; case 'P': put_utf8(out, 0x2029); break;
                case 'x': case 'u': case 'U': {
                    const size_t n = e == 'x' ? 2 : e == 'u' ? 4 : 8;
                    if (i + n > s.size()) throw YamlError{};
                    uint32_t c2 = 0;
                    for (size_t k = 0; k < n; ++k) {
                        const char h = s[i + k];
                        const int d = h >= '0' && h <= '9' ? h - '0' : h >= 'a' && h <= 'f' ? h - 'a' + 10 : h >= 'A' && h <= 'F' ? h - 'A' + 10 : -1;
                        if (d < 0) throw YamlError{};
                        c2 = c2 * 16 + (uint32_t)d;
                    }
                    i += n;
                    put_utf8(out, c2);
                    break;
                }
                default: throw YamlError{};
            }
            continue;
        }
        out += c;
    }
}

std::string rtrim(const std::string& s) { size_t n = s.size(); while (n > 0 && (s[n - 1] == ' ' || s[n - 1] == '\t')) --n; return s.substr(0, n); }

// An inline value: a quoted scalar, [] or {}, or a plain scalar
YValue inline_value(const std::string& text) {
    const std::string t = rtrim(text);
    YValue v;
    if (t == "[]") { v.kind = YValue::Seq; return v; }
    if (t == "{}") { v.kind = YValue::Map; return v; }
    if (!t.empty() && (t[0] == '\'' || t[0] == '"')) {
        size_t i = 0;
        v.kind = YValue::Str; v.text = quoted(t, i);
        if (i != t.size()) throw YamlError{};
        return v;
    }
    if (!t.empty() && (t[0] == '[' || t[0] == '{' || t[0] == '|' || t[0] == '>' || t[0] == '&' || t[0] == '*' || t[0] == '!' ||
                       t[0] == '@' || t[0] == '`' || t[0] == '%')) throw YamlError{};
    return plain_scalar(t);
}

bool is_seq_item(const std::string& t) { return t == "-" || (t.size() >= 2 && t[0] == '-' && t[1] == ' '); }

// Splits "key: value" / "key:" into the key and the value text; false when the line is no mapping entry
bool split_entry(const std::string& t, YValue& key, std::string& rest) {
    size_t i = 0;
    if (!t.empty() && (t[0] == '\'' || t[0] == '"')) {
        key.kind = YValue::Str; key.text = quoted(t, i);
        while (i < t.size() && t[i] == ' ') ++i;
        if (i >= t.size() || t[i] != ':' || (i + 1 < t.size() && t[i + 1] != ' ')) return false;
        rest = i + 1 < t.size() ? t.substr(i + 2) : "";
        return true;
    }
    for (; i < t.size(); ++i)
        if (t[i] == ':' && (i + 1 == t.size() || t[i + 1] == ' ')) {
            key = plain_scalar(rtrim(t.substr(0, i)));
            rest = i + 1 < t.size() ? t.substr(i + 2) : "";
            return true;
        }
    return false;
}

struct YamlReader {
    std::vector<YLine> lines;
    size_t at = 0;

    YValue block(size_t indent) {                         // the node whose first line is lines[at], at this indentation
        return is_seq_item(lines[at].text) ? sequence(indent) : mapping(indent);
    }
    // the value of an entry whose text after "key:" or "-" is empty: a nested block, a sequence at the key's own indentation, or null
    YValue nested(size_t indent, bool allow_same_indent_seq) {
        if (at < lines.size() && lines[at].indent > indent) return block(lines[at].indent);
        if (allow_same_indent_seq && at < lines.size() && lines[at].indent == indent && is_seq_item(lines[at].text)) return sequence(indent);
        return YValue();
    }
    YValue sequence(size_t indent) {
        YValue v; v.kind = YValue::Seq;
        while (at < lines.size() && lines[at].indent == indent && is_seq_item(lines[at].text)) {
            const std::string item = lines[at].text.size() > 2 ? lines[at].text.substr(2) : "";
            size_t lead = 0;
            while (lead < item.size() && item[lead] == ' ') ++lead;
            const std::string body = item.substr(lead);
            YValue key; std::string rest;
            if (body.empty()) { ++at; v.items.push_back(nested(indent, false)); }
            else if (is_seq_item(body) || split_entry(body, key, rest)) {   // a nested node that starts on the item's line
                lines[at].indent = indent + 2 + lead; lines[at].text = body;
                v.items.push_back(block(lines[at].indent));
            } else { ++at; v.items.push_back(inline_value(body)); }
        }
        if (at < lines.size() && lines[at].indent > indent) throw YamlError{};
        return v;
    }
    YValue mapping(size_t indent) {
        YValue v; v.kind = YValue::Map;
        while (at < lines.size() && lines[at].indent == indent && !is_seq_item(lines[at].text)) {
            YValue key; std::string rest;
            if (!split_entry(lines[at].text, key, rest)) throw YamlError{};
            ++at;
            for (size_t x = 0; x < v.items.size(); x += 2)     // serde_yaml refuses a duplicate key
                if (v.items[x].kind == key.kind && v.items[x].text == key.text && v.items[x].b == key.b && v.items[x].kind != YValue::Float) throw YamlError{};
            v.items.push_back(key);
            size_t lead = 0;
            while (lead < rest.size() && rest[lead] == ' ') ++lead;
            v.items.push_back(lead == rest.size() ? nested(indent, true) : inline_value(rest.substr(lead)));
        }
        if (at < lines.size() && lines[at].indent > indent) throw YamlError{};
        return v;
    }
};

// serde_yaml::from_str::<HashMap<String, Value>>: the document must be a mapping with string keys
std::vector<std::pair<std::string, YValue>> load_yaml_map(const std::string& path) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) throw InputError{"Could not read YAML file"};
    std::string text; char buf[1 << 16]; size_t n;
    while ((n = fread(buf, 1, sizeof buf, f)) > 0) text.append(buf, n);
    const bool bad = ferror(f);
    fclose(f);
    if (bad) throw InputError{"Could not read YAML file"};
    YamlReader r;
    size_t a = 0;
    while (a < text.size()) {
        size_t b = text.find('\n', a);
        if (b == std::string::npos) b = text.size();
        std::string line = text.substr(a, b - a);
        if (!line.empty() && line.back() == '\r') line.pop_back();
        a = b + 1;
        size_t ind = 0;
        while (ind < line.size() && line[ind] == ' ') ++ind;
        const std::string body = rtrim(line.substr(ind));
        if (body.empty() || body[0] == '#' || (ind == 0 && body == "---")) continue;
        if (body[0] == '\t') throw InputError{"Failed to parse YAML file"};
        r.lines.push_back({ind, body});
    }
    std::vector<std::pair<std::string, YValue>> out;
    try {
        if (r.lines.empty() || r.lines[0].indent != 0 || is_seq_item(r.lines[0].text)) throw YamlError{};
        if (r.lines.size() == 1 && r.lines[0].text == "{}") return out;
        YValue m = r.mapping(0);
        if (r.at != r.lines.size()) throw YamlError{};
        for (size_t x = 0; x < m.items.size(); x += 2) {
            const YValue& k = m.items[x];
            if (k.kind != YValue::Str && k.kind != YValue::Int && k.kind != YValue::Bool) throw YamlError{};
            out.emplace_back(k.kind == YValue::Bool ? (k.b ? "true" : "false") : k.text, m.items[x + 1]);
        }
    } catch (const YamlError&) { throw InputError{"Failed to parse YAML file"}; }
    return out;
}

std::string format_value(const YValue& v, uint64_t sigfigs) {     // table.rs:158-194
    switch (v.kind) {
        case YValue::Int: return v.text;
        case YValue::Float: return format_float_sigfigs(v.f, sigfigs);
        case YValue::Str: return v.text;
        case YValue::Bool: return v.b ? "true" : "false";
        case YValue::Seq: {
            std::string s = "[";
            for (size_t i = 0; i < v.items.size(); ++i) s += (i ? "," : "") + format_value(v.items[i], sigfigs);
            return s + "]";
        }
        case YValue::Map: {
            std::string s = "{";
            for (size_t i = 0; i < v.items.size(); i += 2) s += (i ? "," : "") + format_value(v.items[i], sigfigs) + ":" + format_value(v.items[i + 1], sigfigs);
            return s + "}";
        }
        default: return "";
    }
}

// ---- the files (table.rs:118-155) ----
bool is_dir(const std::string& p) { struct stat st; return stat(p.c_str(), &st) == 0 && S_ISDIR(st.st_mode); }

std::string join(const std::string& dir, const std::string& name) { return dir.empty() || dir.back() == '/' ? dir + name : dir + "/" + name; }

void visit(const std::string& dir, std::vector<std::string>& out) {     // visit_dirs_for_yaml_files; unreadable entries are skipped
    DIR* d = opendir(dir.c_str());
    if (!d) return;
    std::vector<std::string> names;
    while (dirent* e = readdir(d)) { const std::string n = e->d_name; if (n != "." && n != "..") names.push_back(n); }
    closedir(d);
    for (const std::string& n : names) {
        const std::string p = join(dir, n);
        if (is_dir(p)) visit(p, out);
        else {
            const size_t dot = n.rfind('.');                // Path::extension: none for a name whose only '.' is its first byte
            if (dot != std::string::npos && dot > 0 && n.compare(dot + 1, std::string::npos, "yaml") == 0) out.push_back(p);
        }
    }
}

std::vector<std::string> components(const std::string& p) {    // Path::components for ordering: empty and "." parts drop out
    std::vector<std::string> c;
    size_t a = 0;
    while (a <= p.size()) {
        size_t b = p.find('/', a);
        if (b == std::string::npos) b = p.size();
        const std::string part = p.substr(a, b - a);
        if (!part.empty() && !(part == "." && !c.empty())) c.push_back(part);
        a = b + 1;
    }
    return c;
}

std::string file_name(const std::string& p) { const size_t s = p.rfind('/'); return s == std::string::npos ? p : p.substr(s + 1); }

std::vector<std::string> one_copy(const std::vector<std::string>& files, const std::string& name, bool verbose) {   // get_one_copy_yaml
    std::vector<std::string> found;
    for (const std::string& f : files) if (file_name(f) == name) found.push_back(f);
    if (found.empty() && verbose) fprintf(stderr, "Warning: %s not found\n", name.c_str());
    if (found.size() > 1) throw InputError{"Multiple " + name + " files found"};
    return found;
}

std::vector<std::string> multi_copy(const std::vector<std::string>& files, const std::string& name, bool verbose) {   // get_multi_copy_yaml
    std::vector<std::string> found;
    for (const std::string& f : files) if (file_name(f) == name && f.find("/qc_fail/") == std::string::npos) found.push_back(f);
    if (found.empty() && verbose) fprintf(stderr, "Warning: %s not found\n", name.c_str());
    return found;
}
}  // namespace

std::string table_text(const std::string& autocycler_dir, bool have_dir, const std::string& name, const std::string& fields_text, uint64_t sigfigs,
                       bool verbose) {
    if (sigfigs == 0) throw InputError{"--sigfigs must be 1 or greater"};
    std::vector<std::string> fields;                      // parse_fields (:43-60)
    {
        std::string t;
        for (char c : fields_text) if (c != ' ') t += c;
        size_t a = 0;
        while (true) {
            const size_t b = std::min(t.find(',', a), t.size());
            fields.push_back(t.substr(a, b - a));
            if (b == t.size()) break;
            a = b + 1;
        }
        const std::set<std::string> valid(std::begin(FIELD_NAMES), std::end(FIELD_NAMES));
        for (const std::string& f : fields) if (!valid.count(f)) throw InputError{f + " is not a valid field name"};
    }
    std::string line;
    if (!have_dir) {                                      // print_header (:63-65)
        line = "name";
        for (const std::string& f : fields) line += "\t" + f;
        return line + "\n";
    }
    if (name.find('\t') != std::string::npos) throw InputError{"--name cannot contain tab characters"};
    std::vector<std::string> files;                       // find_all_yaml_files, sorted as PathBuf sorts: component by component
    visit(autocycler_dir, files);
    std::vector<std::pair<std::vector<std::string>, std::string>> keyed;
    for (const std::string& f : files) keyed.emplace_back(components(f), f);
    std::sort(keyed.begin(), keyed.end());
    files.clear();
    for (auto& k : keyed) files.push_back(k.second);

    std::map<std::string, YValue> map;                    // later files overwrite earlier keys (HashMap::extend)
    std::vector<std::string> singles;
    for (const char* f : {"subsample.yaml", "input_assemblies.yaml", "clustering.yaml", "consensus_assembly.yaml"}) {
        const std::vector<std::string> found = one_copy(files, f, verbose);
        if (!found.empty()) singles.push_back(found[0]);
    }
    const std::vector<std::string> untrimmed = multi_copy(files, "1_untrimmed.yaml", verbose), trimmed = multi_copy(files, "2_trimmed.yaml", verbose);
    for (const std::string& p : singles) for (auto& kv : load_yaml_map(p)) map[kv.first] = std::move(kv.second);
    for (const std::vector<std::string>* group : {&untrimmed, &trimmed}) {     // load_multi_yaml_to_map: each key's values, in path order
        std::map<std::string, YValue> combined;
        for (const std::string& p : *group)
            for (auto& kv : load_yaml_map(p)) {
                YValue& s = combined[kv.first];
                s.kind = YValue::Seq;
                s.items.push_back(std::move(kv.second));
            }
        for (auto& kv : combined) map[kv.first] = std::move(kv.second);
    }
    line = name;
    for (const std::string& f : fields) {
        line += "\t";
        const auto it = map.find(f);
        if (it != map.end()) line += format_value(it->second, sigfigs);
    }
    return line + "\n";
}
