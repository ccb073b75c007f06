// `autocycler trim` (trim.rs:36-326): the overlap alignments run on the device in batches (DeviceAlign::overlap_align: fill,
// right-edge maximum and traceback); what is O(k) per alignment — the identity test (:468-475), find_midpoint (:482-507) and the
// hairpin walk (:299-317) — and the graph edits run here, in f64 and u32 exactly as the reference writes them.
#include "host_trim.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <deque>
#include <stdexcept>

#include "commands.h"
#include "host_io.h"

namespace {
const int32_t GAP = 0;                 // trim.rs:32
typedef std::deque<AlignPiece> Alignment;

std::vector<int32_t> reverse_path(const std::vector<int32_t>& p) {     // misc.rs:443-445
    std::vector<int32_t> r(p.size());
    for (size_t x = 0; x < p.size(); ++x) r[x] = -p[p.size() - 1 - x];
    return r;
}

uint32_t weight_of(const std::vector<uint32_t>& w, int32_t u) {
    const uint64_t a = u < 0 ? (uint64_t)(-(int64_t)u) : (uint64_t)u;
    if (a >= w.size()) throw std::runtime_error("unitig " + std::to_string(a) + " has no weight");
    return w[a];
}

struct Pair { const std::vector<int32_t>* a; const std::vector<int32_t>* b; bool skip; };

// One cluster's part of a device round: its pairs, its weight table (by its own unitig numbers) and, after the round, its alignments
struct PairSet {
    std::vector<Pair> pairs;
    const std::vector<uint32_t>* weights;
    TrimStats* stats;
    std::vector<Alignment> out;
};

// sign * (|u| + base): a cluster's unitig number in the batch's concatenated weight table
int32_t rebase(int32_t u, uint64_t base) {
    const uint64_t a = (u < 0 ? (uint64_t)(-(int64_t)u) : (uint64_t)u) + base;
    if (a >= 0x80000000ull) throw RangeError{"unitig " + std::to_string(a) + " of the batch's weight table does not fit 31 bits"};
    return u < 0 ? -(int32_t)a : (int32_t)a;
}
int32_t unbase(int32_t v, uint64_t base) { return v == GAP ? GAP : v < 0 ? v + (int32_t)base : v - (int32_t)base; }

// overlap_alignment (:366-479) for every pair of every set in one device round: the device's traceback, then the identity test.  The
// sets' weight tables are concatenated and each set's unitigs rebased onto its part of it; path equality only compares unitigs of one
// set, so the rebased alignments are the sets' own.
void overlap_alignments(DeviceAlign& device, const std::vector<PairSet*>& sets, double min_identity, uint32_t max_unitigs, AlignBatch& batch) {
    std::vector<int32_t> values;
    std::vector<uint32_t> weights;
    std::vector<OverlapJob> jobs;
    std::vector<uint64_t> base(sets.size());
    for (size_t s = 0; s < sets.size(); ++s) {
        const PairSet& S = *sets[s];
        base[s] = weights.size();
        weights.insert(weights.end(), S.weights->begin(), S.weights->end());
        const size_t first = values.size();
        for (const Pair& p : S.pairs) {
            if (p.a->size() != p.b->size()) throw std::runtime_error("overlap_alignment: paths of different lengths");   // :379
            const uint64_t n = p.a->size();
            if (n > 0x7FFFFFFFull) throw std::runtime_error("paths longer than 2^31 unitigs are not supported");
            OverlapJob J;
            J.n = (uint32_t)n; J.k = (uint32_t)std::min<uint64_t>(max_unitigs, n); J.skip_diagonal = p.skip ? 1 : 0; J.pad = 0;
            J.a_off = values.size(); values.insert(values.end(), p.a->begin(), p.a->end());
            if (p.b == p.a) J.b_off = J.a_off;
            else { J.b_off = values.size(); values.insert(values.end(), p.b->begin(), p.b->end()); }
            jobs.push_back(J);
            S.stats->cells += (uint64_t)J.k * J.k; S.stats->max_window = std::max(S.stats->max_window, J.k); S.stats->max_path = std::max<uint64_t>(S.stats->max_path, n);
            batch.cells += (uint64_t)J.k * J.k;
        }
        for (size_t v = first; v < values.size(); ++v) { weight_of(*S.weights, values[v]); values[v] = rebase(values[v], base[s]); }
        S.stats->rounds += 1; S.stats->jobs += S.pairs.size();
    }
    std::vector<std::vector<AlignPiece>> raw;
    AlignRun run;
    batch.kernel_ms += device.overlap_align(values.data(), values.size(), weights.data(), weights.size(), jobs.data(), (uint32_t)jobs.size(), raw, &run);
    batch.launches += run.launches(); batch.jobs += jobs.size(); batch.buffer_bytes = std::max(batch.buffer_bytes, run.buffer_bytes);
    size_t x = 0;
    for (size_t s = 0; s < sets.size(); ++s) {
        PairSet& S = *sets[s];
        const std::vector<uint32_t>& w = *S.weights;
        S.out.assign(S.pairs.size(), {});
        for (size_t q = 0; q < S.pairs.size(); ++q, ++x) {
            std::vector<AlignPiece>& al = raw[x];
            if (al.empty()) continue;
            for (AlignPiece& p : al) { p.a_unitig = unbase(p.a_unitig, base[s]); p.b_unitig = unbase(p.b_unitig, base[s]); }
            uint32_t a_len = 0, b_len = 0, matches = 0;                       // u32 sums (:468-471)
            for (const AlignPiece& p : al) {
                if (p.a_unitig != GAP) a_len += weight_of(w, p.a_unitig);
                if (p.b_unitig != GAP) b_len += weight_of(w, p.b_unitig);
                if (p.a_unitig == p.b_unitig) matches += weight_of(w, p.a_unitig);
            }
            const double mean_length = ((double)a_len + (double)b_len) / 2.0;
            const double identity = (double)matches / mean_length;
            if (identity < min_identity) continue;
            S.out[q].assign(al.begin(), al.end());
        }
    }
}

size_t find_midpoint(const Alignment& al, const std::vector<uint32_t>& w) {     // :482-507
    uint32_t total = 0;
    for (const AlignPiece& p : al) {
        uint32_t x = 0;
        if (p.a_unitig != GAP) x += weight_of(w, p.a_unitig);
        if (p.b_unitig != GAP) x += weight_of(w, p.b_unitig);
        total += x;
    }
    uint32_t cumulative = 0;
    size_t best_index = 0;
    double best_closeness = 1.0;
    for (size_t i = 0; i < al.size(); ++i) {
        const AlignPiece& p = al[i];
        if (p.a_unitig != GAP) cumulative += weight_of(w, p.a_unitig);
        if (p.b_unitig != GAP) cumulative += weight_of(w, p.b_unitig);
        const double closeness = std::fabs(0.5 - ((double)cumulative / (double)total));
        if (p.a_unitig == p.b_unitig && closeness < best_closeness) { best_index = i; best_closeness = closeness; }
    }
    return best_index;
}

// trim_path_start_end's tail (:291-295)
bool finish_start_end(const std::vector<int32_t>& path, const Alignment& al, const std::vector<uint32_t>& w, std::vector<int32_t>& out) {
    if (al.empty()) return false;
    const size_t mid = find_midpoint(al, w);
    const int32_t start = al[mid].a_index, end = al[mid].b_index;
    if (start < 0 || end < 0 || start > end || (size_t)end > path.size()) throw std::runtime_error("start-end trim: midpoint outside the path");
    out.assign(path.begin() + start, path.begin() + end);
    return true;
}

// trim_path_hairpin_end's walk (:303-316) on the alignment of reverse_path(path) against path
bool finish_hairpin_end(const std::vector<int32_t>& path, Alignment al, std::vector<int32_t>& out) {
    if (al.empty()) return false;
    int32_t end = 0;
    while (!al.empty()) {
        while (!al.empty() && al.front().a_unitig == GAP) al.pop_front();     // trim_gaps_a_front
        while (!al.empty() && al.back().b_unitig == GAP) al.pop_back();       // trim_gaps_b_back
        if (al.empty()) break;
        const AlignPiece back = al.back(); al.pop_back();
        if (al.empty() || back.b_unitig != -al.front().a_unitig) throw std::runtime_error("hairpin trim: back.b_unitig != -front.a_unitig (trim.rs:310)");
        if (back.a_unitig != GAP) end = back.b_index;
        al.pop_front();
    }
    out.assign(path.begin(), path.begin() + end);
    return true;
}

}  // namespace

// median_isize / mad_isize (misc.rs:399-423): integer halving of the two middle values for even counts
int64_t median_i64(std::vector<int64_t> v) {
    if (v.empty()) return 0;
    std::sort(v.begin(), v.end());
    const size_t n = v.size();
    return n % 2 == 0 ? (v[n / 2 - 1] + v[n / 2]) / 2 : v[n / 2];
}
int64_t mad_i64(const std::vector<int64_t>& v) {
    if (v.empty()) return 0;
    const int64_t m = median_i64(v);
    std::vector<int64_t> dev(v.size());
    for (size_t x = 0; x < v.size(); ++x) dev[x] = v[x] > m ? v[x] - m : m - v[x];
    return median_i64(dev);
}

namespace {
uint64_t round_to_usize(double x) {   // (x).round() as usize: half away from zero, negatives and NaN saturate to 0
    const double r = std::round(x);
    if (!(r > 0)) return 0;
    if (r >= 18446744073709551615.0) return UINT64_MAX;
    return (uint64_t)r;
}
}  // namespace

void trim_paths(DeviceAlign& device, TrimMode mode, const std::vector<std::vector<int32_t>>& paths, const std::vector<uint32_t>& weights,
                double min_identity, uint32_t max_unitigs, std::vector<uint8_t>& trimmed, std::vector<std::vector<int32_t>>& out, TrimStats& stats) {
    const size_t N = paths.size();
    trimmed.assign(N, 0); out.assign(N, {});
    std::vector<std::vector<int32_t>> rev(N);
    std::vector<Pair> pairs(N);
    for (size_t x = 0; x < N; ++x) {
        if (mode == TRIM_START_END) pairs[x] = Pair{&paths[x], &paths[x], true};                       // :290
        else {
            rev[x] = reverse_path(paths[x]);
            // hairpin end: reverse_path(path) against path (:301-302); hairpin start is the hairpin end of the reversed path (:322-323),
            // i.e. path against reverse_path(path)
            pairs[x] = mode == TRIM_HAIRPIN_END ? Pair{&rev[x], &paths[x], false} : Pair{&paths[x], &rev[x], false};
        }
    }
    PairSet set{std::move(pairs), &weights, &stats, {}};
    AlignBatch batch;
    overlap_alignments(device, {&set}, min_identity, max_unitigs, batch);
    stats.kernel_ms += batch.kernel_ms;
    const std::vector<Alignment>& al = set.out;
    for (size_t x = 0; x < N; ++x) {
        if (mode == TRIM_START_END) trimmed[x] = finish_start_end(paths[x], al[x], weights, out[x]);
        else if (mode == TRIM_HAIRPIN_END) trimmed[x] = finish_hairpin_end(paths[x], al[x], out[x]);
        else {
            std::vector<int32_t> t;
            trimmed[x] = finish_hairpin_end(rev[x], al[x], t);
            if (trimmed[x]) out[x] = reverse_path(t);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// the graph edits trim needs (unitig_graph.rs:151-174, 547-586)
// ------------------------------------------------------------------------------------------------
void HostGraph::replace_paths(const std::vector<std::vector<UStrand>>& paths) {
    std::vector<uint64_t> off(paths.size() + 1, 0);
    std::vector<UStrand> all;
    for (size_t q = 0; q < paths.size(); ++q) { all.insert(all.end(), paths[q].begin(), paths[q].end()); off[q + 1] = all.size(); }
    own_path_off.swap(off); own_path.swap(all);
    path_off = own_path_off.data(); path = own_path.data(); n_path = own_path.size(); n_seqs = (uint32_t)paths.size();
    fpos_off.clear(); rpos_off.clear(); fpos.clear(); rpos.clear();      // full position lists are not kept through trim's edits
    fixed_ready = false; cands_ready = false;
}

void HostGraph::recalculate_depths() {
    std::vector<double> d(U, 0.0);
    for (uint64_t x = 0; x < n_path; ++x) d[us_index(path[x])] += 1.0;
    std::vector<uint32_t> di(U);
    for (uint32_t u = 0; u < U; ++u) di[u] = (uint32_t)d[u];
    std::vector<uint8_t> ty(U);
    for (uint32_t u = 0; u < U; ++u) ty[u] = type_of(u);
    own_depth_f.swap(d); own_depth.swap(di); own_type.swap(ty);
    depth_f = own_depth_f.data(); depth = own_depth.data(); utype = own_type.data();
}

void HostGraph::remove_zero_depth_unitigs() {
    const uint32_t GONE = 0xFFFFFFFFu;
    std::vector<uint32_t> new_index(U, GONE), old_of;
    for (uint32_t n = 0; n < U; ++n) { const uint32_t u = order[n]; if (depth_of(u) > 0.0) { new_index[u] = (uint32_t)old_of.size(); old_of.push_back(u); } }
    const uint32_t U2 = (uint32_t)old_of.size();
    std::vector<UnitigRec> rec2(U2); std::vector<uint32_t> depth2(U2), number2(U2), order2(U2);
    std::vector<double> depth_f2(U2); std::vector<uint8_t> type2(U2);
    for (uint32_t v = 0; v < U2; ++v) {
        const uint32_t u = old_of[v];
        rec2[v] = rec[u]; depth2[v] = depth[u]; number2[v] = number[u]; depth_f2[v] = depth_of(u); type2[v] = type_of(u); order2[v] = v;
    }
    // delete_dangling_links: every list keeps its order, minus the entries that lead to a removed unitig
    std::vector<uint32_t> next_off2(2 * (size_t)U2 + 1, 0), prev_off2(2 * (size_t)U2 + 1, 0);
    std::vector<UStrand> next2, prev2;
    for (uint32_t v = 0; v < U2; ++v)
        for (uint32_t r = 0; r < 2; ++r) {
            const UStrand s = us_make(old_of[v], r != 0);
            for (uint32_t x = 0; x < next_size(s); ++x) { const UStrand t = next_begin(s)[x]; if (new_index[us_index(t)] != GONE) next2.push_back(us_make(new_index[us_index(t)], us_reverse(t))); }
            next_off2[2 * (size_t)v + r + 1] = (uint32_t)next2.size();
            for (uint32_t x = 0; x < prev_size(s); ++x) { const UStrand t = prev_begin(s)[x]; if (new_index[us_index(t)] != GONE) prev2.push_back(us_make(new_index[us_index(t)], us_reverse(t))); }
            prev_off2[2 * (size_t)v + r + 1] = (uint32_t)prev2.size();
        }
    std::vector<UStrand> path2(n_path);
    for (uint64_t x = 0; x < n_path; ++x) {
        const uint32_t v = new_index[us_index(path[x])];
        if (v == GONE) throw std::runtime_error("remove_zero_depth_unitigs: a path runs through a unitig of depth 0");
        path2[x] = us_make(v, us_reverse(path[x]));
    }
    std::vector<uint64_t> path_off2(path_off, path_off + n_seqs + 1);
    own_rec.swap(rec2); own_depth.swap(depth2); number.swap(number2); order.swap(order2); own_depth_f.swap(depth_f2); own_type.swap(type2);
    own_next_off.swap(next_off2); own_prev_off.swap(prev_off2); own_next.swap(next2); own_prev.swap(prev2);
    own_path.swap(path2); own_path_off.swap(path_off2);
    U = U2; rec = own_rec.data(); depth = own_depth.data(); depth_f = own_depth_f.data(); utype = own_type.data();
    next_off = own_next_off.data(); prev_off = own_prev_off.data(); next = own_next.data(); prev = own_prev.data(); n_links = own_next.size();
    path_off = own_path_off.data(); path = own_path.data();
    fpos_off.clear(); rpos_off.clear(); fpos.clear(); rpos.clear();
    fixed_ready = false; cands_ready = false; first_pass = true;
    check_links();
}

// ------------------------------------------------------------------------------------------------
// trim.rs:43-51
// ------------------------------------------------------------------------------------------------
namespace {
std::string seq_display(const HostSeq& s) {     // sequence.rs:112-135 without the bracketed extras
    return s.filename + " " + s.contig_header.substr(0, s.contig_header.find(' ')) + " (" + std::to_string(s.length) + " bp)";
}
void section(FILE* log, const char* title) { if (log) fprintf(log, "\n%s\n", title); }
}  // namespace

namespace {
// One cluster between the phases of trim_graphs
struct TrimWork {
    TrimCluster* c;
    size_t S = 0;
    uint32_t max_number = 0;
    std::vector<uint32_t> weights, index_of;                   // by unitig number: length before any edit (:44), index in the graph
    std::vector<std::vector<int32_t>> paths, rev, path2, rev2, se_path, hp_path;
    std::vector<uint8_t> se_ok, hp_ok, start_ok;
    PairSet set;
    uint32_t path_length(const std::vector<int32_t>& p) const { uint32_t t = 0; for (int32_t u : p) t += weight_of(weights, u); return t; }
};

// the weights and the paths by unitig number, and round 1: start-end and hairpin start (trim_start_end_overlap, :113-136, and
// trim_harpin_overlap, :139-186)
void trim_prepare(TrimWork& w, uint32_t max_unitigs) {
    HostGraph& g = *w.c->g;
    const size_t S = w.S = w.c->seqs->size();
    if (g.n_seqs != S) throw std::runtime_error("trim: the graph's paths do not match its sequences");
    for (uint32_t u = 0; u < g.U; ++u) w.max_number = std::max(w.max_number, g.number[u]);
    w.weights.assign((size_t)w.max_number + 1, 0);
    w.index_of.assign((size_t)w.max_number + 1, 0xFFFFFFFFu);
    for (uint32_t u = 0; u < g.U; ++u) { w.weights[g.number[u]] = g.rec[u].len; w.index_of[g.number[u]] = u; }
    w.paths.assign(S, {});
    for (size_t q = 0; q < S; ++q)
        for (uint64_t x = g.path_off[q]; x < g.path_off[q + 1]; ++x) { const int32_t num = (int32_t)g.number[us_index(g.path[x])]; w.paths[q].push_back(us_reverse(g.path[x]) ? -num : num); }
    w.se_ok.assign(S, 0); w.hp_ok.assign(S, 0); w.se_path.assign(S, {}); w.hp_path.assign(S, {});
    w.set.weights = &w.weights; w.set.stats = &w.c->stats;
    if (max_unitigs == 0) return;
    w.rev.assign(S, {});
    for (size_t q = 0; q < S; ++q) w.rev[q] = reverse_path(w.paths[q]);
    for (size_t q = 0; q < S; ++q) { w.set.pairs.push_back(Pair{&w.paths[q], &w.paths[q], true}); w.set.pairs.push_back(Pair{&w.paths[q], &w.rev[q], false}); }
}

// round 1's results, and round 2: hairpin end on the hairpin-start results
void trim_round2(TrimWork& w) {
    const size_t S = w.S;
    const std::vector<Alignment> r1 = std::move(w.set.out);
    w.start_ok.assign(S, 0); w.path2.assign(S, {});
    for (size_t q = 0; q < S; ++q) {
        w.se_ok[q] = finish_start_end(w.paths[q], r1[2 * q], w.weights, w.se_path[q]);
        std::vector<int32_t> t;
        w.start_ok[q] = finish_hairpin_end(w.rev[q], r1[2 * q + 1], t);
        w.path2[q] = w.start_ok[q] ? reverse_path(t) : w.paths[q];
    }
    w.rev2.assign(S, {});
    w.set.pairs.clear();
    for (size_t q = 0; q < S; ++q) { w.rev2[q] = reverse_path(w.path2[q]); w.set.pairs.push_back(Pair{&w.rev2[q], &w.path2[q], false}); }
}

// round 2's results and their report
void trim_apply_round2(TrimWork& w) {
    const size_t S = w.S;
    FILE* log = w.c->log;
    const std::vector<HostSeq>& seqs = *w.c->seqs;
    for (size_t q = 0; q < S; ++q) {
        std::vector<int32_t> t;
        const bool end_ok = finish_hairpin_end(w.path2[q], w.set.out[q], t);
        w.hp_ok[q] = w.start_ok[q] || end_ok;
        if (w.hp_ok[q]) w.hp_path[q] = end_ok ? t : w.path2[q];
    }
    if (log) {
        section(log, "Trim start-end overlaps");
        for (size_t q = 0; q < S; ++q)
            if (w.se_ok[q]) fprintf(log, "%s: trimmed to %u bp\n", seq_display(seqs[q]).c_str(), w.path_length(w.se_path[q]));
            else fprintf(log, "%s: not trimmed\n", seq_display(seqs[q]).c_str());
        section(log, "Trim hairpin overlaps");
        for (size_t q = 0; q < S; ++q)
            if (w.hp_ok[q]) fprintf(log, "%s: trimmed to %u bp\n", seq_display(seqs[q]).c_str(), w.path_length(w.hp_path[q]));
            else fprintf(log, "%s: not trimmed\n", seq_display(seqs[q]).c_str());
    }
}

// choose_trim_type, the length outliers and the clean-up
void trim_finish(TrimWork& w, double mad) {
    const size_t S = w.S;
    FILE* log = w.c->log;
    HostGraph& g = *w.c->g;
    std::vector<HostSeq>& seqs = *w.c->seqs;
    std::vector<std::vector<int32_t>>& paths = w.paths;
    // choose_trim_type (:189-226): on a tie, start-end
    const size_t se_count = std::count(w.se_ok.begin(), w.se_ok.end(), 1), hp_count = std::count(w.hp_ok.begin(), w.hp_ok.end(), 1);
    if (se_count > 0 || hp_count > 0) {
        const bool use_se = se_count >= hp_count;
        if (log && use_se && hp_count > 0) fprintf(log, "\nStart-end trimming was more successful than hairpin trimming. Discarding hairpin trimming.\n");
        if (log && !use_se && se_count > 0) fprintf(log, "\nHairpin trimming was more successful than start-end trimming. Discarding start-end trimming.\n");
        for (size_t q = 0; q < S; ++q) {
            if (!(use_se ? w.se_ok[q] : w.hp_ok[q])) continue;
            paths[q] = use_se ? w.se_path[q] : w.hp_path[q];
            seqs[q].length = w.path_length(paths[q]);
        }
    }

    // exclude_outliers_in_length (:229-257)
    std::vector<uint8_t> keep(S, 1);
    if (mad != 0.0) {
        std::vector<int64_t> lengths(S);
        for (size_t q = 0; q < S; ++q) lengths[q] = (int64_t)seqs[q].length;
        const int64_t median = median_i64(lengths), dev = mad_i64(lengths);
        const uint64_t lo = round_to_usize((double)median - ((double)dev * mad)), hi = round_to_usize((double)median + ((double)dev * mad));
        section(log, "Exclude outliers");
        if (log) fprintf(log, "Median sequence length:    %lld bp\nMedian absolute deviation: %lld bp\nAllowed length range:      %llu-%llu bp\n\n",
                         (long long)median, (long long)dev, (unsigned long long)lo, (unsigned long long)hi);
        for (size_t q = 0; q < S; ++q) {
            keep[q] = lo <= seqs[q].length && seqs[q].length <= hi;
            if (log) fprintf(log, "%s: %s\n", seq_display(seqs[q]).c_str(), keep[q] ? "kept" : "excluded");
        }
    }

    // the new paths (through the graph's current unitig indices) of the kept sequences
    std::vector<std::vector<UStrand>> new_paths;
    std::vector<HostSeq> kept;
    for (size_t q = 0; q < S; ++q) {
        if (!keep[q]) continue;
        std::vector<UStrand> p(paths[q].size());
        for (size_t x = 0; x < p.size(); ++x) {
            const int32_t s = paths[q][x];
            const uint32_t num = (uint32_t)(s < 0 ? -s : s);
            if (num > w.max_number || w.index_of[num] == 0xFFFFFFFFu) throw std::runtime_error("unitig " + std::to_string(num) + " not found in unitig index");
            p[x] = us_make(w.index_of[num], s < 0);
        }
        new_paths.push_back(std::move(p));
        kept.push_back(seqs[q]);
    }
    seqs.swap(kept);

    // clean_up_graph (:260-269)
    g.replace_paths(new_paths);
    g.recalculate_depths();
    g.remove_zero_depth_unitigs();
    g.merge_linear_paths(true);
    g.renumber();
    section(log, "Clean graph");
    if (log) fprintf(log, "%u unitig%s, %llu link%s\ntotal length: %llu bp\n\n", g.U, g.U == 1 ? "" : "s", (unsigned long long)g.link_count_single(),
                     g.link_count_single() == 1 ? "" : "s", (unsigned long long)g.total_length());
}
}  // namespace

void trim_graphs(DeviceAlign& device, std::vector<TrimCluster>& clusters, double min_identity, uint32_t max_unitigs, double mad, AlignBatch& batch) {
    std::vector<TrimWork> work(clusters.size());
    std::vector<PairSet*> sets;
    for (size_t c = 0; c < clusters.size(); ++c) { work[c].c = &clusters[c]; trim_prepare(work[c], max_unitigs); sets.push_back(&work[c].set); }
    batch.clusters += (uint32_t)clusters.size();
    if (max_unitigs > 0) {
        overlap_alignments(device, sets, min_identity, max_unitigs, batch);
        for (TrimWork& w : work) trim_round2(w);
        overlap_alignments(device, sets, min_identity, max_unitigs, batch);
        for (TrimWork& w : work) trim_apply_round2(w);
    }
    for (TrimWork& w : work) trim_finish(w, mad);
    if (clusters.size() == 1) clusters[0].stats.kernel_ms = batch.kernel_ms;     // a shared launch's time belongs to no one cluster
}

void trim_graph(HostGraph& g, std::vector<HostSeq>& seqs, DeviceAlign& device, double min_identity, uint32_t max_unitigs, double mad,
                bool verbose, TrimStats& stats) {
    std::vector<TrimCluster> one{TrimCluster{&g, &seqs, verbose ? stderr : nullptr, TrimStats()}};
    AlignBatch batch;
    trim_graphs(device, one, min_identity, max_unitigs, mad, batch);
    stats = one[0].stats;
}

std::string trimmed_metrics_yaml(const std::vector<HostSeq>& seqs) {
    // median_usize / mad_usize (misc.rs:389-415) of the lengths, as u32
    std::vector<int64_t> lengths;
    for (const HostSeq& s : seqs) lengths.push_back((int64_t)s.length);
    const int64_t median = median_i64(lengths), dev = mad_i64(lengths);
    std::string y = "trimmed_cluster_size: " + std::to_string((uint32_t)seqs.size()) + "\n";
    if (seqs.empty()) y += "trimmed_cluster_lengths: []\n";
    else { y += "trimmed_cluster_lengths:\n"; for (const HostSeq& s : seqs) y += "- " + std::to_string(s.length) + "\n"; }
    y += "trimmed_cluster_median: " + std::to_string((uint32_t)median) + "\n";
    y += "trimmed_cluster_mad: " + std::to_string((uint32_t)dev) + "\n";
    return y;
}
