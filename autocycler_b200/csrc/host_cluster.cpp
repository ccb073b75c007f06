// `autocycler cluster` (cluster.rs:30-912) on the host, around the device's distance and UPGMA kernels (DeviceCluster::cluster_distances,
// DeviceCluster::upgma).  The f64 operations are the reference's, in its order, except where the reference's own order is a HashMap's
// (DESIGN.md §12): the balance score sums clusters in ascending number, and a cluster contained in several passed clusters names the
// smallest of them.
#include "host_cluster.h"

#include <algorithm>
#include <charconv>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <map>
#include <set>

#include "host_io.h"
#include "host_trim.h"
#include "commands.h"

namespace {
void fail(const std::string& m) { throw InputError{m}; }

// section_header + explanation (log.rs), without colours, the timestamp or the terminal-width wrapping
void section(bool verbose, const char* title, const char* text) {
    if (verbose) fprintf(stderr, "\n%s\n    %s\n\n", title, text);
}

std::string lower(std::string s) { for (char& c : s) if (c >= 'A' && c <= 'Z') c = (char)(c + 32); return s; }
uint64_t header_weight(const std::string& header, const std::string& key) {   // sequence.rs:97-109
    const std::string low = lower(header);
    for (size_t a = 0; a < low.size();) {
        while (a < low.size() && isspace((unsigned char)low[a])) ++a;
        size_t b = a; while (b < low.size() && !isspace((unsigned char)low[b])) ++b;
        if (b > a && low.compare(a, key.size(), key) == 0 && b - a > key.size()) {
            const std::string v = low.substr(a + key.size(), b - a - key.size());
            const size_t first = v[0] == '+' ? 1 : 0;
            if (v.size() > first && v.find_first_not_of("0123456789", first) == std::string::npos) return strtoull(v.c_str(), nullptr, 10);
        }
        a = b;
    }
    return 1;
}
uint64_t cluster_weight(const HostSeq& s) { return header_weight(s.contig_header, "autocycler_cluster_weight="); }
uint64_t consensus_weight(const HostSeq& s) { return header_weight(s.contig_header, "autocycler_consensus_weight="); }
bool is_trusted(const HostSeq& s) { return lower(s.contig_header).find("autocycler_trusted") != std::string::npos; }
std::string contig_name(const HostSeq& s) { return s.contig_header.substr(0, s.contig_header.find(' ')); }
std::string newick_name(const HostSeq& s) {   // sequence.rs:85-87
    return std::to_string(s.id) + "__" + s.filename + "__" + contig_name(s) + "__" + std::to_string(s.length) + "_bp";
}
std::string display(const HostSeq& s) {       // sequence.rs:112-135
    std::vector<std::string> extras;
    const std::string low = lower(s.contig_header);
    if (low.find("autocycler_trusted") != std::string::npos) extras.push_back("trusted");
    if (low.find("autocycler_ignore") != std::string::npos) extras.push_back("ignored");
    if (cluster_weight(s) != 1) extras.push_back("cluster weight = " + std::to_string(cluster_weight(s)));
    if (consensus_weight(s) != 1) extras.push_back("consensus weight = " + std::to_string(consensus_weight(s)));
    std::string t = s.filename + " " + contig_name(s) + " (" + std::to_string(s.length) + " bp)";
    if (!extras.empty()) { t += " ["; for (size_t i = 0; i < extras.size(); ++i) { if (i) t += ", "; t += extras[i]; } t += "]"; }
    return t;
}

// shortest round-trip digits of v > 0 and the decimal exponent of the first one (v = 0.d1d2... x 10^(point))
void shortest_digits(double v, std::string& digits, int& point) {
    char buf[64];
    const auto r = std::to_chars(buf, buf + sizeof buf, v, std::chars_format::scientific);
    const std::string s(buf, r.ptr);
    const size_t e = s.find('e');
    digits.clear();
    for (size_t i = 0; i < e; ++i) if (s[i] != '.') digits += s[i];
    point = atoi(s.c_str() + e + 1) + 1;
}

// The tree of the merge list (cluster.rs:195-348), indexed by node number; a tip has no children.
struct Tree {
    std::vector<uint32_t> left, right;
    std::vector<double> dist;
    std::vector<uint8_t> exists;
    uint32_t root = 0;
    bool tip(uint32_t u) const { return left[u] == 0; }
    bool has(uint32_t u) const { return u < exists.size() && exists[u]; }
    void tips(uint32_t u, std::vector<uint32_t>& out) const {   // collect_tips (:288-295), left before right
        if (tip(u)) { out.push_back(u); return; }
        tips(left[u], out); tips(right[u], out);
    }
    void collect(uint32_t u, double cutoff, const std::vector<uint16_t>& manual, const std::vector<uint8_t>& manual_below, std::vector<uint32_t>& out) const {
        const bool in_manual = std::binary_search(manual.begin(), manual.end(), (uint16_t)u) && u <= 0xFFFF;
        if (in_manual || (dist[u] <= cutoff && !manual_below[u])) out.push_back(u);         // collect_clusters (:239-247)
        else if (!tip(u)) { collect(left[u], cutoff, manual, manual_below, out); collect(right[u], cutoff, manual, manual_below, out); }
    }
};

bool in_manual(const std::vector<uint16_t>& manual, uint32_t u) { return u <= 0xFFFF && std::binary_search(manual.begin(), manual.end(), (uint16_t)u); }

// has_manual_child (:249-258) of every node, bottom-up
std::vector<uint8_t> manual_below(const Tree& t, const std::vector<uint16_t>& manual) {
    std::vector<uint8_t> hm(t.exists.size(), 0);
    std::vector<std::pair<uint32_t, bool>> st{{t.root, false}};
    while (!st.empty()) {
        auto [u, done] = st.back(); st.pop_back();
        if (t.tip(u)) { hm[u] = in_manual(manual, u); continue; }
        if (!done) { st.push_back({u, true}); st.push_back({t.left[u], false}); st.push_back({t.right[u], false}); continue; }
        hm[u] = in_manual(manual, u) || hm[t.left[u]] || hm[t.right[u]];
    }
    return hm;
}

struct ClusterQC { std::vector<std::string> reasons; double dist = 0; bool pass() const { return reasons.empty(); } };

struct Metrics {       // ClusteringMetrics (metrics.rs:111-183)
    uint32_t pass_clusters = 0, fail_clusters = 0, pass_contigs = 0, fail_contigs = 0;
    double pass_fraction = 0, fail_fraction = 0, balance = 0, tightness = 0, overall = 0;
};

struct Clusterer {
    const Tree& t;
    std::vector<HostSeq>& seqs;
    const std::vector<double>& asym;
    double cutoff; uint64_t min_assemblies;
    std::vector<uint32_t> index_of;            // sequence id -> index in seqs
    std::vector<uint8_t> contains;             // [a * S + b]: d_ab < d_ba && d_ab < cutoff (cluster_is_contained_in_another's test)
    std::vector<uint32_t> filename_id; uint32_t n_filenames = 0;
    std::vector<uint8_t> trusted; std::vector<uint64_t> cweight;

    Clusterer(const Tree& t_, std::vector<HostSeq>& s, const std::vector<double>& d, double c, uint64_t m) : t(t_), seqs(s), asym(d), cutoff(c), min_assemblies(m) {
        const size_t S = seqs.size();
        uint32_t max_id = 0;
        for (auto& q : seqs) max_id = std::max<uint32_t>(max_id, q.id);
        index_of.assign(max_id + 1, 0);
        for (size_t i = 0; i < S; ++i) index_of[seqs[i].id] = (uint32_t)i;
        contains.assign(S * S, 0);
        for (size_t a = 0; a < S; ++a)
            for (size_t b = 0; b < S; ++b) { const double ab = asym[a * S + b], ba = asym[b * S + a]; contains[a * S + b] = ab < ba && ab < cutoff; }
        std::map<std::string, uint32_t> fid;
        for (auto& q : seqs) if (!fid.count(q.filename)) { uint32_t k = (uint32_t)fid.size(); fid[q.filename] = k; }
        n_filenames = (uint32_t)fid.size();
        for (auto& q : seqs) { filename_id.push_back(fid[q.filename]); trusted.push_back(is_trusted(q)); cweight.push_back(cluster_weight(q)); }
    }

    // qc_clusters (:511-570): assigns cluster numbers to the sequences and returns the QC of clusters 1..C (index c - 1)
    std::vector<ClusterQC> qc(const std::vector<uint32_t>& nodes, const std::vector<uint16_t>& manual) {
        const size_t S = seqs.size();
        std::vector<ClusterQC> q;
        for (uint32_t n : nodes) {
            if (!t.has(n)) fail("clustering tree does not contain a node with id " + std::to_string(n));
            const uint16_t c = (uint16_t)(q.size() + 1);
            std::vector<uint32_t> tips; t.tips(n, tips);
            for (uint32_t id : tips) seqs[index_of[id]].cluster = c;
            ClusterQC x; x.dist = t.dist[n] * 2.0;                                      // max_pairwise_distance (:208-217)
            if (!manual.empty() && !in_manual(manual, n)) x.reasons.push_back("not included in manual clusters");
            q.push_back(x);
        }
        const size_t C = q.size();
        // reorder_clusters (:881-902): median length descending, ties by the old number
        std::vector<std::vector<int64_t>> lengths(C);
        for (auto& s : seqs) lengths[s.cluster - 1].push_back((int64_t)s.length);
        std::vector<std::pair<int64_t, uint32_t>> order;
        for (uint32_t c = 0; c < C; ++c) order.push_back({median_i64(lengths[c]), c});
        std::sort(order.begin(), order.end(), [](auto& x, auto& y) { return x.first != y.first ? x.first > y.first : x.second < y.second; });
        std::vector<uint16_t> old_to_new(C);
        std::vector<ClusterQC> r(C);
        for (uint32_t k = 0; k < C; ++k) { old_to_new[order[k].second] = (uint16_t)(k + 1); r[k] = q[order[k].second]; }
        for (auto& s : seqs) s.cluster = old_to_new[s.cluster - 1];
        if (!manual.empty()) return r;
        std::vector<std::vector<uint32_t>> members(C);
        for (size_t i = 0; i < S; ++i) members[seqs[i].cluster - 1].push_back((uint32_t)i);
        for (uint32_t c = 0; c < C; ++c) {
            std::map<uint32_t, uint64_t> w;                                             // cluster_assembly_count (:573-585)
            bool tr = false;
            for (uint32_t i : members[c]) { uint64_t& x = w[filename_id[i]]; x = std::max(x, cweight[i]); tr = tr || trusted[i]; }
            uint64_t count = 0; for (auto& kv : w) count += kv.second;
            if (count < min_assemblies && !tr) r[c].reasons.push_back("present in too few assemblies");
        }
        // cluster_is_contained_in_another (:692-723): contained pairs between every two clusters, counted once
        std::vector<uint64_t> pair_count((size_t)C * C, 0);
        for (size_t a = 0; a < S; ++a) {
            const size_t ca = seqs[a].cluster - 1;
            for (size_t b = 0; b < S; ++b) if (contains[a * S + b]) ++pair_count[ca * C + seqs[b].cluster - 1];
        }
        for (uint32_t c = 0; c < C; ++c) {
            bool tr = false; for (uint32_t i : members[c]) tr = tr || trusted[i];
            for (uint32_t p = 0; p < C; ++p) {
                if (p == c || !r[p].pass()) continue;
                const double frac = (double)pair_count[(size_t)c * C + p] / (double)((uint64_t)members[c].size() * members[p].size());
                if (frac > 0.5) { if (!tr) r[c].reasons.push_back("contained within cluster " + std::to_string(p + 1)); break; }
            }
        }
        return r;
    }

    Metrics metrics(const std::vector<ClusterQC>& q) const {     // clustering_metrics (:852-878)
        Metrics m;
        std::vector<double> pass_dist;
        for (auto& x : q) { if (x.pass()) { ++m.pass_clusters; pass_dist.push_back(x.dist); } else ++m.fail_clusters; }
        for (auto& s : seqs) { if (q[s.cluster - 1].pass()) ++m.pass_contigs; else ++m.fail_contigs; }
        const uint32_t total = m.pass_contigs + m.fail_contigs;
        if (total > 0) { m.pass_fraction = (double)m.pass_contigs / (double)total; m.fail_fraction = (double)m.fail_contigs / (double)total; }
        // calculate_balance: the per-filename scores are 0 or 1 (exact sums); clusters are summed in ascending number
        const size_t C = q.size();
        std::vector<std::vector<uint32_t>> counts(C, std::vector<uint32_t>(n_filenames, 0));
        std::vector<uint64_t> size(C, 0);
        for (size_t i = 0; i < seqs.size(); ++i) { ++counts[seqs[i].cluster - 1][filename_id[i]]; ++size[seqs[i].cluster - 1]; }
        double weighted = 0.0, total_weight = 0.0;
        for (size_t c = 0; c < C; ++c) {
            if (size[c] == 0) continue;
            double ones = 0.0; for (uint32_t f = 0; f < n_filenames; ++f) ones += counts[c][f] == 1 ? 1.0 : 0.0;
            const double score = ones / (double)n_filenames;
            weighted += score * (double)size[c];
            total_weight += (double)size[c];
        }
        m.balance = weighted / total_weight;
        if (pass_dist.empty()) m.tightness = 0.0;
        else { double s = 0.0; for (double d : pass_dist) s += 1.0 - std::sqrt(d); m.tightness = s / (double)pass_dist.size(); }
        m.overall = (m.balance + m.tightness) / 2.0;
        return m;
    }

    // split_clusters (:311-335)
    std::vector<std::vector<uint32_t>> splits(const std::vector<uint32_t>& clusters) const {
        std::vector<std::vector<uint32_t>> res;
        for (uint32_t c : clusters) {
            if (t.tip(c)) continue;
            std::vector<uint32_t> alt;
            for (uint32_t o : clusters) if (o != c) alt.push_back(o);
            alt.push_back(t.left[c]); alt.push_back(t.right[c]);
            std::sort(alt.begin(), alt.end());
            res.push_back(alt);
        }
        std::sort(res.begin(), res.end());
        return res;
    }

    std::vector<uint32_t> refine(const std::vector<uint32_t>& start) {     // refine_auto_clusters (:607-630)
        std::vector<uint32_t> best = start;
        double best_score = metrics(qc(best, {})).overall;
        for (bool improved = true; improved;) {
            improved = false;
            for (const auto& alt : splits(best)) {
                const double s = metrics(qc(alt, {})).overall;
                if (s > best_score) { best = alt; best_score = s; improved = true; }
            }
        }
        return best;
    }
};

std::string tree_newick(const Tree& t, uint32_t u, const std::vector<HostSeq>& seqs, const std::vector<uint32_t>& index_of) {   // :381-392
    if (t.tip(u)) return newick_name(seqs[index_of[u]]);
    const uint32_t l = t.left[u], r = t.right[u];
    return "(" + tree_newick(t, l, seqs, index_of) + ":" + rust_display_f64(t.dist[u] - t.dist[l]) + "," + tree_newick(t, r, seqs, index_of) + ":" +
           rust_display_f64(t.dist[u] - t.dist[r]) + ")" + std::to_string(u);
}

std::string untrimmed_yaml(const std::vector<uint64_t>& lengths, double dist) {   // UntrimmedClusterMetrics (metrics.rs:186-205)
    std::vector<int64_t> v(lengths.begin(), lengths.end());
    std::string y = "untrimmed_cluster_size: " + std::to_string(lengths.size()) + "\n";
    if (lengths.empty()) y += "untrimmed_cluster_lengths: []\n";
    else { y += "untrimmed_cluster_lengths:\n"; for (uint64_t x : lengths) y += "- " + std::to_string(x) + "\n"; }
    y += "untrimmed_cluster_median: " + std::to_string((uint32_t)median_i64(v)) + "\n";
    y += "untrimmed_cluster_mad: " + std::to_string((uint32_t)mad_i64(v)) + "\n";
    return y + "untrimmed_cluster_distance: " + yaml_f64(dist) + "\n";
}

// the lines of `gfa` without the P lines of the given sequence ids (filter_gfa_lines, :809-822)
std::string filter_paths(const std::string& gfa, const std::vector<uint8_t>& drop) {
    std::string out;
    out.reserve(gfa.size());
    for (size_t a = 0; a < gfa.size();) {
        size_t b = gfa.find('\n', a);
        b = b == std::string::npos ? gfa.size() : b + 1;
        bool keep = true;
        if (b - a > 2 && gfa[a] == 'P' && gfa[a + 1] == '\t') {
            size_t e = a + 2; uint32_t id = 0; bool num = true;
            while (e < b && gfa[e] != '\t' && gfa[e] != '\n' && gfa[e] != '\r') { num = num && isdigit((unsigned char)gfa[e]) && (id = id * 10 + (gfa[e] - '0')) <= 0xFFFF; ++e; }
            keep = !(num && e > a + 2 && id < drop.size() && drop[id]);
        }
        if (keep) out.append(gfa, a, b - a);
        a = b;
    }
    return out;
}
}  // namespace

uint64_t sequence_consensus_weight(const HostSeq& s) { return consensus_weight(s); }

std::string rust_display_f64(double v) {
    if (std::isnan(v)) return "NaN";
    if (std::isinf(v)) return v > 0 ? "inf" : "-inf";
    const std::string sign = std::signbit(v) ? "-" : "";
    if (v == 0) return sign + "0";
    std::string d; int point;
    shortest_digits(std::fabs(v), d, point);
    if (point <= 0) return sign + "0." + std::string(-point, '0') + d;
    if ((size_t)point >= d.size()) return sign + d + std::string(point - d.size(), '0');
    return sign + d.substr(0, point) + "." + d.substr(point);
}

std::string yaml_f64(double v) {
    if (std::isnan(v)) return ".nan";
    if (std::isinf(v)) return v > 0 ? ".inf" : "-.inf";
    const std::string sign = std::signbit(v) ? "-" : "";
    if (v == 0) return sign + "0.0";
    std::string d; int kk;
    shortest_digits(std::fabs(v), d, kk);
    const int len = (int)d.size(), k = kk - len;                    // v = d x 10^k, kk = the position of the decimal point
    if (k >= 0 && kk <= 16) return sign + d + std::string(k, '0') + ".0";
    if (kk > 0 && kk <= 16) return sign + d.substr(0, kk) + "." + d.substr(kk);
    if (kk > -5 && kk <= 0) return sign + "0." + std::string(-kk, '0') + d;
    if (len == 1) return sign + d + "e" + std::to_string(kk - 1);
    return sign + d.substr(0, 1) + "." + d.substr(1) + "e" + std::to_string(kk - 1);
}

std::string format_float(double v) {
    char buf[400];
    snprintf(buf, sizeof buf, "%.6f", v);
    std::string s = buf;
    if (s.find('.') == std::string::npos) return s;
    while (!s.empty() && s.back() == '0') s.pop_back();
    if (!s.empty() && s.back() == '.') s.pop_back();
    return s;
}

std::vector<uint16_t> parse_manual_clusters(const std::string& text) {
    std::string t;
    for (char c : text) if (c != ' ') t += c;
    std::vector<uint16_t> out;
    for (size_t a = 0;;) {
        size_t b = t.find(',', a);
        const std::string s = t.substr(a, b == std::string::npos ? std::string::npos : b - a);
        const size_t first = !s.empty() && s[0] == '+' ? 1 : 0;           // str::parse::<u16>
        bool okay = s.size() > first && s.find_first_not_of("0123456789", first) == std::string::npos && s.size() - first <= 10;
        const uint64_t v = okay ? strtoull(s.c_str() + first, nullptr, 10) : 0;
        if (!okay || v > 0xFFFF) fail("failed to parse '" + s + "' as a node number");
        out.push_back((uint16_t)v);
        if (b == std::string::npos) break;
        a = b + 1;
    }
    std::sort(out.begin(), out.end());
    return out;
}

std::string distance_matrix_text(const std::vector<HostSeq>& seqs, const double* d) {
    const size_t S = seqs.size();
    std::string text = std::to_string(S) + "\n";
    for (size_t a = 0; a < S; ++a) {
        text += display(seqs[a]);
        for (size_t b = 0; b < S; ++b) { char buf[400]; snprintf(buf, sizeof buf, "\t%.8f", d[a * S + b]); text += buf; }
        text += "\n";
    }
    return text;
}

void cluster_graph(const std::string& gfa, const HostGraph& g, std::vector<HostSeq>& seqs, DeviceCluster& device, double cutoff, int64_t min_assemblies_opt,
                   const std::vector<uint16_t>& manual, uint32_t max_contigs, const std::string& out_dir, bool verbose, ClusterResult& out, ClusterStats& st) {
    const size_t S = seqs.size();
    std::set<std::string> files;
    for (auto& s : seqs) files.insert(s.filename);
    uint64_t min_assemblies;                                           // set_min_assemblies (:645-661)
    if (min_assemblies_opt >= 0) min_assemblies = (uint64_t)min_assemblies_opt;
    else if (files.size() == 1) min_assemblies = 1;
    else min_assemblies = std::max<uint64_t>(2, (files.size() + 2) / 4);
    if (verbose) {                                                     // print_settings (:98-114)
        fprintf(stderr, "  --cutoff %s\n", format_float(cutoff).c_str());
        if (min_assemblies_opt < 0) fprintf(stderr, "  --min_assemblies %llu (automatically set)\n", (unsigned long long)min_assemblies);
        else fprintf(stderr, "  --min_assemblies %llu\n", (unsigned long long)min_assemblies);
        fprintf(stderr, "  --max_contigs %u\n", max_contigs);
        if (!manual.empty()) { std::string m; for (size_t i = 0; i < manual.size(); ++i) m += (i ? "," : "") + std::to_string(manual[i]); fprintf(stderr, "  --manual %s\n", m.c_str()); }
        fprintf(stderr, "\n");
    }
    if (S == 0) fail("no sequences found in input_assemblies.gfa");   // check_sequence_count (:117-129)
    const double mean = (double)S / (double)files.size();
    if (mean > (double)max_contigs) {
        char buf[64]; snprintf(buf, sizeof buf, "%.1f", mean);
        fail(std::string("the mean number of contigs per input assembly (") + buf + ") exceeds the allowed threshold (" + std::to_string(max_contigs) +
             "). Are your input assemblies fragmented or contaminated?");
    }
    // pairwise_contig_distances + make_symmetrical_distances on the device; the symmetric matrix stays there for UPGMA
    std::vector<uint32_t> len(g.U);
    for (uint32_t u = 0; u < g.U; ++u) len[u] = g.rec[u].len;
    std::vector<double> asym(S * S);
    st = ClusterStats(); st.n_seqs = (uint32_t)S;
    st.distance_ms = device.cluster_distances(g.path, g.path_off, (uint32_t)S, len.data(), g.U, asym.data());
    // two sequences whose unitig sets are both empty have no distance (0 / 0): the reference's UPGMA cannot finish on them either
    for (size_t a = 0; a < S; ++a)
        for (size_t b = a + 1; b < S; ++b)
            if (asym[a * S + b] != asym[a * S + b] && asym[b * S + a] != asym[b * S + a])
                fail("the distance between sequences " + std::to_string(seqs[a].id) + " and " + std::to_string(seqs[b].id) + " is not a number (their paths have no length)");
    out.phylip = distance_matrix_text(seqs, asym.data());
    if (verbose) {
        section(verbose, "Pairwise distances", "Every pairwise distance between contigs is calculated based on the similarity of their paths through the graph.");
        fprintf(stderr, "%zu sequences, %zu total pairwise distances\n\nSaving distance matrix:\n  %s/pairwise_distances.phylip\n\n", S, S * S, out_dir.c_str());
        section(verbose, "Clustering sequences", "Contigs are organised into a tree using UPGMA. Then clusters are defined from the tree using the distance cutoff.");
    }
    // UPGMA over the sequences in ascending id order (the reference's sorted keys)
    std::vector<uint32_t> by_id(S);
    for (size_t i = 0; i < S; ++i) by_id[i] = (uint32_t)i;
    std::sort(by_id.begin(), by_id.end(), [&](uint32_t x, uint32_t y) { return seqs[x].id < seqs[y].id; });
    std::vector<uint32_t> ids(S);
    bool ordered = true;
    for (size_t i = 0; i < S; ++i) { ids[i] = seqs[by_id[i]].id; ordered = ordered && by_id[i] == i; }
    std::vector<UpgmaMerge> merges(S ? S - 1 : 0);
    if (ordered) st.upgma_ms = device.upgma(nullptr, (uint32_t)S, ids.data(), merges.data());
    else {
        std::vector<double> sym(S * S);
        for (size_t x = 0; x < S; ++x)
            for (size_t y = 0; y < S; ++y) { const double ab = asym[by_id[x] * S + by_id[y]], ba = asym[by_id[y] * S + by_id[x]]; sym[x * S + y] = (ab != ab || ab < ba) ? ba : ab; }
        st.upgma_ms = device.upgma(sym.data(), (uint32_t)S, ids.data(), merges.data());
    }
    Tree t;
    const uint32_t n_nodes = ids.back() + (uint32_t)S;
    t.left.assign(n_nodes, 0); t.right.assign(n_nodes, 0); t.dist.assign(n_nodes, 0.0); t.exists.assign(n_nodes, 0);
    for (uint32_t id : ids) t.exists[id] = 1;
    t.root = ids[0];
    for (auto& m : merges) { t.left[m.node] = m.left; t.right[m.node] = m.right; t.dist[m.node] = m.dist; t.exists[m.node] = 1; t.root = m.node; }
    if (t.dist[t.root] > 0.5) {                                        // normalise_tree (:483-494)
        const double f = 0.5 / t.dist[t.root];
        for (uint32_t u = 0; u < n_nodes; ++u) if (t.exists[u]) t.dist[u] *= f;
    }
    Clusterer cl(t, seqs, asym, cutoff, min_assemblies);
    const std::string nw = tree_newick(t, t.root, seqs, cl.index_of);  // save_tree_to_newick (:363-378)
    out.newick = t.dist[t.root] < 0.5 ? "(" + nw + ":" + rust_display_f64(0.5 - t.dist[t.root]) + ");\n" : nw + ";\n";
    if (verbose) fprintf(stderr, "Saving clustering tree:\n  %s/clustering.newick\n\n", out_dir.c_str());
    // generate_clusters (:497-508)
    std::vector<uint32_t> nodes;
    const std::vector<uint8_t> hm = manual_below(t, manual);
    if (manual.empty()) {
        t.collect(t.root, cutoff / 2.0, manual, hm, nodes);
        std::sort(nodes.begin(), nodes.end());
        nodes = cl.refine(nodes);
    } else {
        for (uint32_t u = 0; u < n_nodes; ++u)                           // check_consistency (:260-271)
            if (t.exists[u] && !t.tip(u) && in_manual(manual, u) && (hm[t.left[u]] || hm[t.right[u]])) fail("manual clusters cannot be nested");
        t.collect(t.root, cutoff / 2.0, manual, hm, nodes);
        std::sort(nodes.begin(), nodes.end());
    }
    const std::vector<ClusterQC> q = cl.qc(nodes, manual);
    const size_t C = q.size();
    out.seq_cluster.resize(S);
    for (size_t i = 0; i < S; ++i) out.seq_cluster[i] = seqs[i].cluster;
    out.cluster_pass.assign(C, 0); out.cluster_gfa.assign(C, ""); out.cluster_yaml.assign(C, "");
    const auto t0 = std::chrono::steady_clock::now();
    for (int pass_round = 1; pass_round >= 0; --pass_round)            // save_qc_pass_clusters, then save_qc_fail_clusters (:726-791)
        for (size_t c = 0; c < C; ++c) {
            if (q[c].pass() != (pass_round == 1)) continue;
            out.cluster_pass[c] = q[c].pass();
            if (verbose) fprintf(stderr, "Cluster %03zu:\n", c + 1);
            std::vector<uint64_t> lengths;
            std::vector<uint8_t> drop(cl.index_of.size(), 0);
            std::vector<HostSeq> members;
            for (auto& s : seqs) {
                if (s.cluster == c + 1) { if (verbose) fprintf(stderr, "  %s\n", display(s).c_str()); lengths.push_back(s.length); members.push_back(s); }
                else drop[s.id] = 1;
            }
            if (verbose) {
                if (lengths.size() > 1) fprintf(stderr, "  cluster distance: %s\n", format_float(q[c].dist).c_str());
                if (q[c].pass()) fprintf(stderr, "  passed QC\n");
                for (auto& r : q[c].reasons) fprintf(stderr, "  failed QC: %s\n", r.c_str());
            }
            // save_cluster_gfa (:794-806): the other clusters' paths dropped, depths recounted, empty unitigs removed, linear paths merged
            const std::string text = filter_paths(gfa, drop);
            HostGraph cg;
            std::vector<HostSeq> loaded;
            cg.load_gfa(text.data(), text.size(), loaded);
            cg.recalculate_depths();
            cg.remove_zero_depth_unitigs();
            cg.merge_linear_paths(true);
            cg.gfa_text(members, out.cluster_gfa[c]);
            out.cluster_yaml[c] = untrimmed_yaml(lengths, q[c].dist);
            if (verbose) fprintf(stderr, "\n");
        }
    st.cluster_gfa_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    // save_data_to_tsv (:832-849)
    out.tsv = "node_name\tpassing_clusters\tall_clusters\tsequence_id\tfile_name\tcontig_name\tlength\ttrusted\tcluster_weight\tconsensus_weight\n";
    for (auto& s : seqs) {
        const bool p = q[s.cluster - 1].pass();
        out.tsv += newick_name(s) + "\t" + (p ? std::to_string(s.cluster) : "none") + "\t" + std::to_string(s.cluster) + "\t" + std::to_string(s.id) + "\t" +
                   s.filename + "\t" + contig_name(s) + "\t" + std::to_string(s.length) + "\t" + (is_trusted(s) ? "true" : "false") + "\t" +
                   std::to_string(cluster_weight(s)) + "\t" + std::to_string(consensus_weight(s)) + "\n";
    }
    const Metrics m = cl.metrics(q);
    out.yaml = "pass_cluster_count: " + std::to_string(m.pass_clusters) + "\nfail_cluster_count: " + std::to_string(m.fail_clusters) +
               "\npass_contig_count: " + std::to_string(m.pass_contigs) + "\nfail_contig_count: " + std::to_string(m.fail_contigs) +
               "\npass_contig_fraction: " + yaml_f64(m.pass_fraction) + "\nfail_contig_fraction: " + yaml_f64(m.fail_fraction) +
               "\ncluster_balance_score: " + yaml_f64(m.balance) + "\ncluster_tightness_score: " + yaml_f64(m.tightness) +
               "\noverall_clustering_score: " + yaml_f64(m.overall) + "\n";
    st.pass_clusters = m.pass_clusters; st.fail_clusters = m.fail_clusters;
}
