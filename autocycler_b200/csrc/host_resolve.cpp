// `autocycler resolve` (resolve.rs:31-514): anchors, bridges, ambiguity and culling, and the graph edits that apply the bridges, on the
// host; the one step whose cost grows quadratically — global_alignment_distance between every pair of a bridge's paths (:430-462) — runs
// on the device (DeviceAlign::bridge_distances).  `autocycler combine` (combine.rs:90-137) works on loaded graphs alone.
//
// The graph edits work on per-strand link lists (the reference's forward_next / reverse_next / forward_prev / reverse_prev vectors, in
// their order), and the host graph's CSR is rebuilt once from them (HostGraph::replace_unitigs) for merge_linear_paths, renumber_unitigs
// and the GFA text.
#include "host_resolve.h"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <map>
#include <set>
#include <stdexcept>
#include <unordered_map>

#include "host_cluster.h"
#include "host_edit.h"
#include "commands.h"
#include "host_io.h"

namespace {
typedef std::vector<int32_t> Path;

Path reverse_path(const Path& p) {     // misc.rs:443-445
    Path r(p.size());
    for (size_t x = 0; x < p.size(); ++x) r[x] = -p[p.size() - 1 - x];
    return r;
}
uint32_t abs_u32(int32_t u) { return u < 0 ? (uint32_t)(-(int64_t)u) : (uint32_t)u; }
inline char complement(char c) { return c == 'A' ? 'T' : c == 'C' ? 'G' : c == 'G' ? 'C' : c == 'T' ? 'A' : c; }
}  // namespace

// ------------------------------------------------------------------------------------------------
// Bridge::new: the best path of every bridge
// ------------------------------------------------------------------------------------------------
void bridge_best_paths(DeviceAlign& device, std::vector<BridgeSet>& sets, AlignBatch& batch) {
    // distinct paths per group (first appearance order) and their multiplicities; every set's unitigs rebased onto its part of the
    // concatenated weight table, sign * (|u| + base): a job only compares the paths of one set
    struct JobRef { uint32_t s, g, p, q; };
    struct SetWork {
        std::vector<std::vector<uint32_t>> which;          // group entry -> distinct index
        std::vector<std::vector<const Path*>> distinct;
        std::vector<std::vector<uint32_t>> mult;
    };
    std::vector<SetWork> work(sets.size());
    std::vector<int32_t> values;
    std::vector<uint32_t> weights;
    std::vector<BridgeJob> jobs;
    std::vector<JobRef> refs;
    for (size_t s = 0; s < sets.size(); ++s) {
        const std::vector<std::vector<Path>>& groups = *sets[s].groups;
        const std::vector<uint32_t>& w = *sets[s].weights;
        ResolveStats& stats = *sets[s].stats;
        SetWork& W = work[s];
        const uint64_t base = weights.size();
        weights.insert(weights.end(), w.begin(), w.end());
        const size_t G = groups.size();
        W.which.assign(G, {}); W.distinct.assign(G, {}); W.mult.assign(G, {});
        std::vector<std::vector<uint64_t>> offset(G);
        for (size_t g = 0; g < G; ++g) {
            std::map<Path, uint32_t> seen;
            for (const Path& p : groups[g]) {
                for (int32_t u : p) if (u == 0 || abs_u32(u) >= w.size()) throw std::runtime_error("unitig " + std::to_string(u) + " has no weight");
                stats.longest_path = std::max<uint64_t>(stats.longest_path, p.size());
                auto it = seen.find(p);
                if (it == seen.end()) {
                    it = seen.emplace(p, (uint32_t)W.distinct[g].size()).first;
                    W.distinct[g].push_back(&p); W.mult[g].push_back(0);
                    offset[g].push_back(values.size());
                    for (int32_t u : p) {
                        const uint64_t a = abs_u32(u) + base;
                        if (a >= 0x80000000ull) throw RangeError{"unitig " + std::to_string(a) + " of the batch's weight table does not fit 31 bits"};
                        values.push_back(u < 0 ? -(int32_t)a : (int32_t)a);
                    }
                }
                W.which[g].push_back(it->second); W.mult[g][it->second] += 1;
            }
            const uint32_t K = (uint32_t)W.distinct[g].size();
            for (uint32_t p = 0; p < K; ++p)
                for (uint32_t q = p + 1; q < K; ++q) {
                    // the shorter path on the rows (D is symmetric bit for bit, DESIGN.md §13)
                    const bool swap = W.distinct[g][q]->size() < W.distinct[g][p]->size();
                    const uint32_t r = swap ? q : p, c = swap ? p : q;
                    const uint64_t n = W.distinct[g][r]->size(), m = W.distinct[g][c]->size();
                    if (m > 0x7FFFFFFFull) throw std::runtime_error("paths longer than 2^31 unitigs are not supported");
                    jobs.push_back(BridgeJob{offset[g][r], offset[g][c], (uint32_t)n, (uint32_t)m});
                    refs.push_back(JobRef{(uint32_t)s, (uint32_t)g, p, q});
                    stats.cells += n * m; stats.jobs += 1;
                    batch.cells += n * m;
                }
        }
    }
    std::vector<uint32_t> dist(jobs.size());
    if (jobs.size() > 0xFFFFFFFFull) throw std::runtime_error("too many distance jobs");
    AlignRun run;
    batch.kernel_ms += device.bridge_distances(values.data(), values.size(), weights.data(), weights.size(), jobs.data(), (uint32_t)jobs.size(), dist.data(), &run);
    batch.launches += run.launches(); batch.jobs += jobs.size(); batch.buffer_bytes = std::max(batch.buffer_bytes, run.buffer_bytes);
    if (sets.size() == 1) {               // a shared launch's split and time belong to no one set
        ResolveStats& stats = *sets[0].stats;
        stats.shared_jobs += run.shared_jobs; stats.hbm_jobs += run.hbm_jobs; stats.kernel_ms += batch.kernel_ms;
    }
    // total(p) = sum over the other distinct paths q of mult(q) * D(p, q), mod 2^32 (copies of p itself add D(p, p) = 0)
    std::vector<std::vector<std::vector<uint32_t>>> dtotal(sets.size());
    for (size_t s = 0; s < sets.size(); ++s) {
        dtotal[s].resize(work[s].distinct.size());
        for (size_t g = 0; g < work[s].distinct.size(); ++g) dtotal[s][g].assign(work[s].distinct[g].size(), 0u);
    }
    for (size_t x = 0; x < refs.size(); ++x) {
        const JobRef& r = refs[x];
        const std::vector<std::vector<uint32_t>>& mult = work[r.s].mult;
        dtotal[r.s][r.g][r.p] += mult[r.g][r.q] * dist[x];
        dtotal[r.s][r.g][r.q] += mult[r.g][r.p] * dist[x];
    }
    // the reference's selection loop over the original order (:440-453): a copy of a path has the same total and never replaces an
    // equal best, so the selected path is the one the all-pairs loop selects
    for (size_t s = 0; s < sets.size(); ++s) {
        const std::vector<std::vector<Path>>& groups = *sets[s].groups;
        const size_t G = groups.size();
        sets[s].totals.assign(G, {}); sets[s].best.assign(G, {});
        for (size_t g = 0; g < G; ++g) {
            uint32_t best_total = 0xFFFFFFFFu;
            const Path* b = nullptr;
            static const Path empty;
            for (size_t x = 0; x < groups[g].size(); ++x) {
                const uint32_t total = dtotal[s][g][work[s].which[g][x]];
                sets[s].totals[g].push_back(total);
                const Path& cur = groups[g][x];
                if (total < best_total || (total == best_total && cur < (b ? *b : empty))) { best_total = total; b = &cur; }
            }
            if (b) sets[s].best[g] = *b;
        }
    }
}

void bridge_best_paths(DeviceAlign& device, const std::vector<std::vector<Path>>& groups, const std::vector<uint32_t>& weights,
                       std::vector<std::vector<uint32_t>>& totals, std::vector<std::vector<int32_t>>& best, ResolveStats& stats) {
    std::vector<BridgeSet> one{BridgeSet{&groups, &weights, &stats, {}, {}}};
    AlignBatch batch;
    bridge_best_paths(device, one, batch);
    totals = std::move(one[0].totals); best = std::move(one[0].best);
}

// ------------------------------------------------------------------------------------------------
// the graph resolve edits
// ------------------------------------------------------------------------------------------------
namespace {
struct Bridge {
    int32_t start, end;
    std::vector<Path> all_paths;       // the trimmed paths, duplicates included
    Path best_path;
    bool conflicting = false;
    int32_t rev_start() const { return -end; }
    int32_t rev_end() const { return -start; }
    size_t depth() const { return all_paths.size(); }
};
// Ord for Bridge (:506-514)
bool bridge_less(const Bridge& a, const Bridge& b) {
    if (abs_u32(a.start) != abs_u32(b.start)) return abs_u32(a.start) < abs_u32(b.start);
    if (a.start != b.start) return a.start > b.start;
    if (abs_u32(a.end) != abs_u32(b.end)) return abs_u32(a.end) < abs_u32(b.end);
    if (a.end != b.end) return a.end > b.end;
    return a.best_path < b.best_path;
}

// determine_ambiguity (:193-220): start and rev_start share one map, end and rev_end the other
size_t determine_ambiguity(std::vector<Bridge>& bridges) {
    std::unordered_map<int32_t, uint32_t> sc, ec;
    for (const Bridge& b : bridges) { sc[b.start] += 1; sc[b.rev_start()] += 1; ec[b.end] += 1; ec[b.rev_end()] += 1; }
    size_t n = 0;
    for (Bridge& b : bridges) {
        b.conflicting = sc[b.start] > 1 || sc[b.rev_start()] > 1 || ec[b.end] > 1 || ec[b.rev_end()] > 1;
        n += b.conflicting;
    }
    return n;
}

// cull_ambiguity (:285-313) in incremental form.  The literal loop removes the first conflicting bridge by (depth, Ord) and recomputes
// every flag.  A bridge's flag depends only on the counts of its four keys, and removing a bridge lowers the counts of its own four
// keys; a flag can only clear when one of its keys' counts falls to 1 or 0.  So the conflicting set is kept ordered, and only the
// bridges of a key whose count has just dropped below 2 are looked at again (each key at most once): the same bridges go in the same
// order, without the quadratic recomputation.
size_t cull_ambiguity(std::vector<Bridge>& bridges, FILE* log) {
    const size_t B = bridges.size();
    std::unordered_map<int32_t, uint32_t> sc, ec;
    std::unordered_map<int32_t, std::vector<uint32_t>> s_members, e_members;
    for (uint32_t x = 0; x < B; ++x) {
        const Bridge& b = bridges[x];
        sc[b.start] += 1; sc[b.rev_start()] += 1; ec[b.end] += 1; ec[b.rev_end()] += 1;
        s_members[b.start].push_back(x); if (b.rev_start() != b.start) s_members[b.rev_start()].push_back(x);
        e_members[b.end].push_back(x); if (b.rev_end() != b.end) e_members[b.rev_end()].push_back(x);
    }
    auto cull_less = [&](uint32_t a, uint32_t b) {
        if (bridges[a].depth() != bridges[b].depth()) return bridges[a].depth() < bridges[b].depth();
        return bridge_less(bridges[a], bridges[b]);
    };
    std::set<uint32_t, decltype(cull_less)> ambi(cull_less);
    std::vector<uint8_t> alive(B, 1);
    auto flag = [&](const Bridge& b) { return sc[b.start] > 1 || sc[b.rev_start()] > 1 || ec[b.end] > 1 || ec[b.rev_end()] > 1; };
    for (uint32_t x = 0; x < B; ++x) if (bridges[x].conflicting) ambi.insert(x);
    size_t culled = 0;
    if (ambi.empty()) return 0;
    if (log) fprintf(log, "\nCulling conflicting bridges\nCulled bridges:\n");
    while (!ambi.empty()) {
        const uint32_t c = *ambi.begin();
        ambi.erase(ambi.begin());
        alive[c] = 0; ++culled;
        const Bridge& b = bridges[c];
        if (log) fprintf(log, "  %d -> %d (%zux)\n", b.start, b.end, b.depth());
        std::vector<const std::vector<uint32_t>*> recheck;
        auto drop = [&](std::unordered_map<int32_t, uint32_t>& counts, std::unordered_map<int32_t, std::vector<uint32_t>>& members, int32_t key) {
            const uint32_t before = counts[key]--;
            if (before >= 2 && before - 1 < 2) recheck.push_back(&members[key]);
        };
        drop(sc, s_members, b.start); drop(sc, s_members, b.rev_start()); drop(ec, e_members, b.end); drop(ec, e_members, b.rev_end());
        for (const std::vector<uint32_t>* list : recheck)
            for (uint32_t y : *list)
                if (alive[y] && bridges[y].conflicting && !flag(bridges[y])) { bridges[y].conflicting = false; ambi.erase(y); }
    }
    std::vector<Bridge> kept;
    for (uint32_t x = 0; x < B; ++x) if (alive[x]) kept.push_back(std::move(bridges[x]));
    bridges.swap(kept);
    if (log) fprintf(log, "\n%zu conflicting bridge%s culled\n\n", culled, culled == 1 ? "" : "s");
    return culled;
}

// apply_bridges (:223-251)
void apply_bridges(EditGraph& G, const std::vector<Bridge>& bridges, double bridge_depth) {
    for (const Bridge& b : bridges) {
        if (b.conflicting) continue;
        const UStrand s = G.strand(b.start), e = G.strand(b.end);
        G.delete_outgoing_links(s);
        G.delete_incoming_links(e);
        if (b.best_path.empty()) { G.create_link(s, e); continue; }
        std::string bridge_seq;                       // get_sequence_from_path_signed
        for (int32_t u : b.best_path) {
            const UStrand t = G.strand(u);
            const std::string& f = G.seq[us_index(t)];
            if (!us_reverse(t)) bridge_seq += f;
            else for (size_t j = f.size(); j-- > 0;) bridge_seq += complement(f[j]);
        }
        const uint32_t num = G.max_number + 1;        // max_unitig_number() + 1
        const uint32_t i = G.add_unitig(num, std::move(bridge_seq), bridge_depth, 2);
        for (const Path& p : b.all_paths)             // reduce_depths (:261-270)
            for (int32_t u : p) { double& d = G.depth[us_index(G.strand(u))]; d -= 1.0; if (d < 0.0) d = 0.0; }
        G.create_link(s, us_make(i, false));
        G.create_link(us_make(i, false), e);
    }
    G.prune();
}

void section(FILE* log, const char* title) { if (log) fprintf(log, "\n%s\n", title); }
void graph_info(FILE* log, const HostGraph& g) {
    if (log) fprintf(log, "%u unitig%s, %llu link%s\ntotal length: %llu bp\n\n", g.U, g.U == 1 ? "" : "s", (unsigned long long)g.link_count_single(),
                         g.link_count_single() == 1 ? "" : "s", (unsigned long long)g.total_length());
}
}  // namespace

void HostGraph::replace_unitigs(const std::vector<uint32_t>& numbers, const std::vector<std::string>& seqs, const std::vector<double>& depths,
                                const std::vector<uint8_t>& types, const std::vector<std::vector<UStrand>>& next_lists,
                                const std::vector<std::vector<UStrand>>& prev_lists) {
    const uint32_t n = (uint32_t)numbers.size();
    uint64_t bytes = 0;
    for (const std::string& s : seqs) bytes += s.size() + 2 * AC_SEQ_SLACK;
    own_rec.assign(n, UnitigRec{}); own_depth.assign(n, 0); own_depth_f.assign(depths.begin(), depths.end()); own_type.assign(types.begin(), types.end());
    number = numbers; order.resize(n);
    arena_overflow.assign(bytes + bytes / 4 + (1u << 16), 0);
    arena = arena_overflow.data(); arena_cap = arena_overflow.size(); arena_used = 0;
    for (uint32_t i = 0; i < n; ++i) {
        UnitigRec& r = own_rec[i];
        r.seq_off = arena_used + AC_SEQ_SLACK; r.len = (uint32_t)seqs[i].size(); r.room_before = r.room_after = AC_SEQ_SLACK; r.flags = 0;
        r.min_fpos = r.min_rpos = 0xFFFFFFFFu;        // positions were cleared (:225)
        memcpy(arena + r.seq_off, seqs[i].data(), seqs[i].size());
        arena_used = r.seq_off + r.len + AC_SEQ_SLACK;
        const double d = depths[i];
        own_depth[i] = (d >= 0 && d <= 4294967295.0) ? (uint32_t)d : 0;
        order[i] = i;
    }
    U = n;
    own_next_off.assign(2 * (size_t)U + 1, 0); own_prev_off.assign(2 * (size_t)U + 1, 0); own_next.clear(); own_prev.clear();
    for (size_t s = 0; s < 2 * (size_t)U; ++s) {
        own_next.insert(own_next.end(), next_lists[s].begin(), next_lists[s].end()); own_next_off[s + 1] = (uint32_t)own_next.size();
        own_prev.insert(own_prev.end(), prev_lists[s].begin(), prev_lists[s].end()); own_prev_off[s + 1] = (uint32_t)own_prev.size();
    }
    own_path.clear(); own_path_off.assign(1, 0);
    rec = own_rec.data(); depth = own_depth.data(); depth_f = own_depth_f.data(); utype = own_type.data();
    next_off = own_next_off.data(); prev_off = own_prev_off.data(); next = own_next.data(); prev = own_prev.data(); n_links = own_next.size();
    path_off = own_path_off.data(); path = own_path.data(); n_path = 0; n_seqs = 0;
    fpos_off.clear(); rpos_off.clear(); fpos.clear(); rpos.clear();
    fixed_ready = false; cands_ready = false; first_pass = true; spec_from_device = false;
    check_links();
}

namespace {
// One cluster between the phases of resolve_texts
struct ResolveWork {
    ResolveCluster* c;
    HostGraph g;
    std::vector<HostSeq> seqs;
    EditGraph loaded;
    std::vector<uint32_t> weights;                        // by unitig number: its length
    std::vector<std::pair<int32_t, int32_t>> keys;        // per bridge: its (start, end)
    std::vector<std::vector<Path>> groups;                // per bridge: its trimmed paths
};

// loading, anchors and the bridges' paths
void resolve_prepare(ResolveWork& w) {
    FILE* log = w.c->log;
    ResolveStats& stats = w.c->stats;
    stats = ResolveStats();
    HostGraph& g = w.g;
    std::vector<HostSeq>& seqs = w.seqs;
    g.load_gfa(w.c->text->data(), w.c->text->size(), seqs);
    section(log, "Loading graph");
    graph_info(log, g);
    EditGraph& loaded = w.loaded;
    loaded.from(g);
    const size_t S = seqs.size();
    std::vector<Path> seq_path(S);
    std::vector<uint32_t> pos(g.U);
    for (uint32_t n = 0; n < g.U; ++n) pos[g.order[n]] = n;
    for (size_t q = 0; q < S; ++q)
        for (uint64_t x = g.path_off[q]; x < g.path_off[q + 1]; ++x) { const int32_t num = (int32_t)g.number[us_index(g.path[x])]; seq_path[q].push_back(us_reverse(g.path[x]) ? -num : num); }

    // find_anchor_unitigs (:134-163): the sorted seq ids of a unitig's forward_positions (one per occurrence in a path, either strand)
    // equal the sorted ids of all sequences; listed in segment order
    std::vector<uint16_t> all_ids;
    for (const HostSeq& s : seqs) all_ids.push_back(s.id);
    std::sort(all_ids.begin(), all_ids.end());
    std::vector<std::vector<uint16_t>> occ(g.U);
    for (size_t q = 0; q < S; ++q) for (uint64_t x = g.path_off[q]; x < g.path_off[q + 1]; ++x) occ[pos[us_index(g.path[x])]].push_back(seqs[q].id);
    std::vector<uint32_t> anchors;
    std::vector<uint8_t> is_anchor_num((size_t)loaded.max_number + 1, 0);
    for (uint32_t i = 0; i < g.U; ++i) {
        std::sort(occ[i].begin(), occ[i].end());
        if (occ[i] == all_ids) { loaded.type[i] = 1; anchors.push_back(loaded.number[i]); is_anchor_num[loaded.number[i]] = 1; }
    }
    stats.anchors = (uint32_t)anchors.size();
    section(log, "Finding anchor unitigs");
    if (log) fprintf(log, "%zu anchor unitig%s found\n\n", anchors.size(), anchors.size() == 1 ? "" : "s");

    // create_bridges (:166-190): every sequence path consensus_weight times, anchor-to-anchor segments (no wrap-around) in the greater of
    // their two orientations, grouped by (first, last) in order of appearance
    w.weights.assign((size_t)loaded.max_number + 1, 0);
    for (uint32_t i = 0; i < g.U; ++i) w.weights[loaded.number[i]] = (uint32_t)loaded.seq[i].size();
    std::map<std::pair<int32_t, int32_t>, uint32_t> group_of;
    for (size_t q = 0; q < S; ++q) {
        const uint64_t wt = sequence_consensus_weight(seqs[q]);
        if (log) fprintf(log, "%s %s (%llu bp) consensus weight = %llu\n", seqs[q].filename.c_str(), seqs[q].contig_header.substr(0, seqs[q].contig_header.find(' ')).c_str(),
                         (unsigned long long)seqs[q].length, (unsigned long long)wt);
        const Path& p = seq_path[q];
        std::vector<Path> segs;
        size_t last = 0; bool have_last = false;
        for (size_t i = 0; i < p.size(); ++i) {
            const uint32_t a = abs_u32(p[i]);
            if (a >= is_anchor_num.size() || !is_anchor_num[a]) continue;
            if (have_last) {
                Path f(p.begin() + last, p.begin() + i + 1), r = reverse_path(f);
                segs.push_back(f > r ? std::move(f) : std::move(r));
            }
            last = i; have_last = true;
        }
        for (uint64_t c = 0; c < wt; ++c)
            for (const Path& sgm : segs) {
                const std::pair<int32_t, int32_t> key(sgm.front(), sgm.back());
                auto it = group_of.find(key);
                if (it == group_of.end()) { it = group_of.emplace(key, (uint32_t)w.groups.size()).first; w.groups.emplace_back(); w.keys.push_back(key); }
                w.groups[it->second].emplace_back(sgm.begin() + 1, sgm.end() - 1);     // Bridge::new drops the start and the end (:432-437)
            }
    }
}

// the bridges with their best paths, ambiguity, both passes and the three texts.  shared: the distances ran in a launch with other
// clusters, so the report leaves the kernel time out.
void resolve_finish(ResolveWork& w, std::vector<Path>& best, bool shared) {
    FILE* log = w.c->log;
    ResolveStats& stats = w.c->stats;
    ResolveResult& out = w.c->out;
    const EditGraph& loaded = w.loaded;
    std::vector<Bridge> bridges(w.groups.size());
    for (size_t x = 0; x < w.groups.size(); ++x) {
        bridges[x].start = w.keys[x].first; bridges[x].end = w.keys[x].second;
        bridges[x].all_paths = std::move(w.groups[x]); bridges[x].best_path = std::move(best[x]);
    }
    std::sort(bridges.begin(), bridges.end(), bridge_less);
    const double bridge_depth = (double)w.seqs.size();   // sequences.len(), not the weighted count
    stats.conflicting_bridges = (uint32_t)determine_ambiguity(bridges);
    stats.unique_bridges = (uint32_t)(bridges.size() - stats.conflicting_bridges);
    section(log, "Building bridges");
    if (log && shared) fprintf(log, "     Unique bridges: %u\nConflicting bridges: %u\n(%llu distance jobs, %llu DP cells)\n\n", stats.unique_bridges,
                               stats.conflicting_bridges, (unsigned long long)stats.jobs, (unsigned long long)stats.cells);
    else if (log) fprintf(log, "     Unique bridges: %u\nConflicting bridges: %u\n(%llu distance jobs, %llu DP cells, distance kernels %.2f ms)\n\n", stats.unique_bridges,
                          stats.conflicting_bridges, (unsigned long long)stats.jobs, (unsigned long long)stats.cells, (double)stats.kernel_ms);

    // first pass: the unique bridges, 3_bridged.gfa, merge, 4_merged.gfa
    section(log, "Applying unique bridges");
    const std::vector<HostSeq> none;
    EditGraph G = loaded;
    apply_bridges(G, bridges, bridge_depth);
    HostGraph h;
    h.k = w.g.k;
    G.to(h);
    h.gfa_text(none, out.bridged);
    h.merge_linear_paths(false);
    graph_info(log, h);
    h.renumber();
    h.gfa_text(none, out.merged);

    // culling, and the second pass on the graph as loaded (the same anchors marked) when anything was culled
    const size_t culled = cull_ambiguity(bridges, log);
    stats.culled_bridges = (uint32_t)culled;
    if (culled > 0) {
        section(log, "Applying final bridges");
        EditGraph G2 = loaded;
        apply_bridges(G2, bridges, bridge_depth);
        HostGraph h2;
        h2.k = w.g.k;
        G2.to(h2);
        h2.merge_linear_paths(false);
        graph_info(log, h2);
        h2.renumber();
        h2.gfa_text(none, out.final_gfa, true);
    } else {
        if (log && !bridges.empty()) fprintf(log, "All bridges were unique, no culling necessary.\n\n");
        h.gfa_text(none, out.final_gfa, true);
    }
}
}  // namespace

void resolve_texts(DeviceAlign& device, std::vector<ResolveCluster>& clusters, AlignBatch& batch) {
    std::vector<ResolveWork> work(clusters.size());
    std::vector<BridgeSet> sets;
    for (size_t c = 0; c < clusters.size(); ++c) {
        work[c].c = &clusters[c];
        resolve_prepare(work[c]);
        sets.push_back(BridgeSet{&work[c].groups, &work[c].weights, &clusters[c].stats, {}, {}});
    }
    batch.clusters += (uint32_t)clusters.size();
    bridge_best_paths(device, sets, batch);
    for (size_t c = 0; c < clusters.size(); ++c) resolve_finish(work[c], sets[c].best, clusters.size() > 1);
}

void resolve_text(const std::string& trimmed_gfa, DeviceAlign& device, bool verbose, ResolveResult& out, ResolveStats& stats) {
    std::vector<ResolveCluster> one{ResolveCluster{&trimmed_gfa, verbose ? stderr : nullptr, {}, {}}};
    AlignBatch batch;
    resolve_texts(device, one, batch);
    out = std::move(one[0].out); stats = one[0].stats;
}

// ------------------------------------------------------------------------------------------------
// combine (combine.rs:90-137)
// ------------------------------------------------------------------------------------------------
void combine_texts(const std::vector<std::string>& gfas, const std::vector<std::string>& names, bool verbose, std::string& gfa, std::string& fasta,
                   std::string& yaml) {
    gfa = "H\tVN:Z:1.0\n"; fasta.clear();
    uint64_t bases = 0; uint32_t unitigs = 0; bool fully_resolved = true;
    std::string clusters;
    uint32_t offset = 0;
    for (size_t f = 0; f < gfas.size(); ++f) {
        HostGraph g;
        std::vector<HostSeq> seqs;
        g.load_gfa(gfas[f].data(), gfas[f].size(), seqs);
        const uint32_t U = g.U;
        auto only = [&](UStrand s, uint32_t u, bool rev) { return g.next_size(s) == 1 && g.next_begin(s)[0] == us_make(u, rev); };
        std::string topology;                          // unitig_graph.rs:527-545
        if (U == 0) topology = "empty";
        else if (U > 1) topology = "fragmented";
        else if (g.n_links == 0) topology = "linear-open-open";
        else if (g.is_isolated_and_circular(0)) topology = "circular";
        else {
            const bool hs = only(us_make(0, true), 0, false), he = only(us_make(0, false), 0, true);
            const bool os = g.next_size(us_make(0, true)) == 0, oe = g.next_size(us_make(0, false)) == 0;
            topology = hs && he ? "linear-hairpin-hairpin" : (hs && oe) || (os && he) ? "linear-open-hairpin" : "other";
        }
        if (verbose) fprintf(stderr, "%s\n%u unitig%s, %llu link%s (%s)\ntotal length: %llu bp\n\n", f < names.size() ? names[f].c_str() : "", U, U == 1 ? "" : "s",
                             (unsigned long long)g.link_count_single(), g.link_count_single() == 1 ? "" : "s", topology.c_str(), (unsigned long long)g.total_length());
        uint32_t max_number = 0;
        char tmp[400];
        for (uint32_t n = 0; n < U; ++n) {
            const uint32_t u = g.order[n];
            max_number = std::max(max_number, g.number[u]);
            const std::string num = std::to_string(g.number[u] + offset), seq(g.seq_ptr(u), g.rec[u].len);
            const uint8_t t = g.type_of(u);
            const char* colour = t == 1 ? "\tCL:Z:forestgreen" : t == 2 ? "\tCL:Z:pink" : t == 3 ? "\tCL:Z:steelblue" : "\tCL:Z:orangered";
            gfa += "S\t" + num + "\t" + seq + "\tDP:f:" + std::string(tmp, gfa_depth_text(tmp, g.depth_of(u))) + colour + "\n";
            fasta += ">" + num + " length=" + std::to_string(g.rec[u].len) +
                     (g.is_isolated_and_circular(u) ? " circular=true topology=circular" : g.is_isolated_and_linear(u) ? " circular=false topology=linear" : "") +
                     "\n" + seq + "\n";
        }
        for (uint32_t n = 0; n < U; ++n) {             // get_links_for_gfa(offset): forward_next, then reverse_next
            const uint32_t u = g.order[n];
            for (uint32_t r = 0; r < 2; ++r) {
                const UStrand s = us_make(u, r != 0);
                for (uint32_t x = 0; x < g.next_size(s); ++x) {
                    const UStrand t = g.next_begin(s)[x];
                    gfa += "L\t" + std::to_string(g.number[u] + offset) + (r ? "\t-\t" : "\t+\t") + std::to_string(g.number[us_index(t)] + offset) +
                           (us_reverse(t) ? "\t-" : "\t+") + "\t0M\n";
                }
            }
        }
        offset += max_number;
        const uint64_t length = g.total_length();
        bases += length; unitigs += U;
        clusters += "- length: " + std::to_string(length) + "\n  unitigs: " + std::to_string(U) + "\n  topology: " + topology + "\n";
        if (U > 1) fully_resolved = false;
    }
    yaml = "consensus_assembly_bases: " + std::to_string(bases) + "\nconsensus_assembly_unitigs: " + std::to_string(unitigs) +
           "\nconsensus_assembly_fully_resolved: " + (fully_resolved ? "true" : "false") + "\nconsensus_assembly_clusters:" +
           (clusters.empty() ? std::string(" []\n") : "\n" + clusters);
}
