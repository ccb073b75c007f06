// A unitig graph as the reference's graph edits see it: unitigs in list order, each with its forward_next / reverse_next and
// forward_prev / reverse_prev vectors in their order (unitig.rs:30-45).  resolve's bridges (host_resolve.cpp) and clean's removals and
// duplications (host_clean.cpp) edit it; the host graph's CSR is rebuilt once from it (HostGraph::replace_unitigs) for
// merge_linear_paths, renumber_unitigs and the GFA text.
#pragma once
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "host_graph.h"

struct EditGraph {
    std::vector<uint32_t> number;
    std::vector<std::string> seq;
    std::vector<double> depth;
    std::vector<uint8_t> type;                        // 0 Other, 1 Anchor, 2 Bridge, 3 Consentig
    std::vector<std::vector<UStrand>> nx, pv;         // [2 i + reverse]: forward_next / reverse_next, forward_prev / reverse_prev
    std::unordered_map<uint32_t, uint32_t> index;     // unitig_index: number -> position
    uint32_t max_number = 0;
    std::vector<uint32_t> visits;                     // forward_positions.len(): the sequence path steps through each unitig

    void from(const HostGraph& g) {
        const uint32_t U = g.U;
        std::vector<uint32_t> pos(U);
        for (uint32_t n = 0; n < U; ++n) pos[g.order[n]] = n;
        number.resize(U); seq.resize(U); depth.resize(U); type.resize(U); nx.assign(2 * (size_t)U, {}); pv.assign(2 * (size_t)U, {});
        index.clear(); max_number = 0; visits.assign(U, 0);
        for (uint64_t x = 0; x < g.n_path; ++x) visits[pos[us_index(g.path[x])]] += 1;
        auto map = [&](UStrand s) { return us_make(pos[us_index(s)], us_reverse(s)); };
        for (uint32_t n = 0; n < U; ++n) {
            const uint32_t u = g.order[n];
            number[n] = g.number[u]; seq[n].assign(g.seq_ptr(u), g.rec[u].len); depth[n] = g.depth_of(u); type[n] = g.type_of(u);
            for (uint32_t r = 0; r < 2; ++r) {
                const UStrand s = us_make(u, r != 0);
                for (uint32_t x = 0; x < g.next_size(s); ++x) nx[2 * (size_t)n + r].push_back(map(g.next_begin(s)[x]));
                for (uint32_t x = 0; x < g.prev_size(s); ++x) pv[2 * (size_t)n + r].push_back(map(g.prev_begin(s)[x]));
            }
            index[number[n]] = n;                     // build_unitig_index: the last unitig with a number wins
            max_number = std::max(max_number, number[n]);
        }
    }
    UStrand strand(int32_t s) const {
        const uint32_t a = s < 0 ? (uint32_t)(-(int64_t)s) : (uint32_t)s;
        const auto it = index.find(a);
        if (it == index.end()) throw std::runtime_error("unitig " + std::to_string(a) + " not found in unitig index");
        return us_make(it->second, s < 0);
    }
    void delete_one_way(UStrand s, UStrand e) {       // unitig_graph.rs:826-865: every matching entry, the others keep their order
        std::vector<UStrand>& a = nx[s]; a.erase(std::remove(a.begin(), a.end(), e), a.end());
        std::vector<UStrand>& b = pv[e]; b.erase(std::remove(b.begin(), b.end(), s), b.end());
    }
    void delete_link(UStrand s, UStrand e) { delete_one_way(s, e); delete_one_way(us_flip(e), us_flip(s)); }
    void delete_outgoing_links(UStrand s) { const std::vector<UStrand> snap = nx[s]; for (UStrand e : snap) delete_link(s, e); }
    void delete_incoming_links(UStrand e) { const std::vector<UStrand> snap = pv[e]; for (UStrand s : snap) delete_link(s, e); }
    void create_one_way(UStrand s, UStrand e) { nx[s].push_back(e); pv[e].push_back(s); }
    void create_link(UStrand s, UStrand e) { create_one_way(s, e); if (s != us_flip(e)) create_one_way(us_flip(e), us_flip(s)); }   // :867-872
    uint32_t add_unitig(uint32_t num, std::string&& s, double d, uint8_t t) {
        const uint32_t i = (uint32_t)number.size();
        number.push_back(num); seq.push_back(std::move(s)); depth.push_back(d); type.push_back(t); visits.push_back(0);
        nx.resize(nx.size() + 2); pv.resize(pv.size() + 2);
        index[num] = i; max_number = std::max(max_number, num);
        return i;
    }
    // Vec::retain over the unitigs, then delete_dangling_links (unitig_graph.rs:547-564) and build_unitig_index: the kept unitigs keep
    // their order, and every list keeps its order minus the entries that lead to a removed unitig
    void retain(const std::vector<uint8_t>& keep) {
        const uint32_t U = (uint32_t)number.size(), NONE = 0xFFFFFFFFu;
        std::vector<uint32_t> new_index(U, NONE);
        uint32_t kept = 0;
        for (uint32_t u = 0; u < U; ++u) if (keep[u]) new_index[u] = kept++;
        EditGraph out;
        for (uint32_t u = 0; u < U; ++u) {
            if (new_index[u] == NONE) continue;
            out.number.push_back(number[u]); out.seq.push_back(std::move(seq[u])); out.depth.push_back(depth[u]); out.type.push_back(type[u]);
            out.visits.push_back(visits[u]);
            for (size_t r = 0; r < 2; ++r) {
                std::vector<UStrand> a, b;
                for (UStrand t : nx[2 * (size_t)u + r]) if (new_index[us_index(t)] != NONE) a.push_back(us_make(new_index[us_index(t)], us_reverse(t)));
                for (UStrand t : pv[2 * (size_t)u + r]) if (new_index[us_index(t)] != NONE) b.push_back(us_make(new_index[us_index(t)], us_reverse(t)));
                out.nx.push_back(std::move(a)); out.pv.push_back(std::move(b));
            }
        }
        for (uint32_t i = 0; i < kept; ++i) { out.index[out.number[i]] = i; out.max_number = std::max(out.max_number, out.number[i]); }
        *this = std::move(out);
    }
    // connected_components (:905-919) without an anchor, then remove_zero_depth_unitigs (depth > 0.0), both with delete_dangling_links
    void prune() {
        const uint32_t U = (uint32_t)number.size(), NONE = 0xFFFFFFFFu;
        std::vector<uint32_t> comp(U, NONE), stack;
        std::vector<uint8_t> comp_has_anchor;
        for (uint32_t s = 0; s < U; ++s) {
            if (comp[s] != NONE) continue;
            const uint32_t c = (uint32_t)comp_has_anchor.size();
            comp_has_anchor.push_back(0);
            comp[s] = c; stack.assign(1, s);
            while (!stack.empty()) {
                const uint32_t u = stack.back(); stack.pop_back();
                if (type[u] == 1) comp_has_anchor[c] = 1;
                for (size_t l = 2 * (size_t)u; l < 2 * (size_t)u + 2; ++l)
                    for (const std::vector<UStrand>* list : {&nx[l], &pv[l]})
                        for (UStrand t : *list) if (comp[us_index(t)] == NONE) { comp[us_index(t)] = c; stack.push_back(us_index(t)); }
            }
        }
        std::vector<uint8_t> keep(U);
        for (uint32_t u = 0; u < U; ++u) keep[u] = comp_has_anchor[comp[u]] && depth[u] > 0.0;
        retain(keep);
    }
    void to(HostGraph& g) const { g.replace_unitigs(number, seq, depth, type, nx, pv); }
};
