// `autocycler polish` on the host (see host_polish.h and DESIGN.md §22).
#include "host_polish.h"

#include <algorithm>
#include <chrono>
#include <stdexcept>

#include "host_depth.h"
#include "host_genome_size.h"
#include "host_qv.h"
#include "host_subsample.h"

namespace {
double ms_since(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

bool acgt(char b) { return b == 'A' || b == 'C' || b == 'G' || b == 'T'; }
uint32_t code_of(char b) { return b == 'A' ? 0 : b == 'C' ? 1 : b == 'G' ? 2 : 3; }
const char* const BASES = "ACGT";

// One round's contigs as the device packs them, and the device's mask of their unsupported windows.
struct Packed {
    std::string bytes;
    std::vector<uint64_t> off, len, woff;    // per contig: first byte, bytes (junction bases included), first packed word (n + 1 values)
    std::vector<uint32_t> mask;
    uint64_t windows = 0, unsupported = 0;
};

void evaluate(DevicePolish& dev, DeviceSpectrum& spec, const std::vector<FastaRecord>& recs, uint32_t k, uint32_t t, Packed& p, PolishResult& out) {
    auto t0 = std::chrono::steady_clock::now();
    p = Packed();
    p.woff.push_back(0);
    for (const FastaRecord& r : recs) {
        p.off.push_back(p.bytes.size());
        p.windows += pack_contig(r, k, p.bytes);
        p.len.push_back(p.bytes.size() - p.off.back());
        p.woff.push_back(p.woff.back() + p.len.back() / 32 + 1);
    }
    p.mask.assign(p.woff.back(), 0);
    out.host_ms += ms_since(t0);
    dev.windows(spec, (const uint8_t*)p.bytes.data(), p.len.data(), (uint32_t)recs.size(), p.windows, t, p.mask.data(), &out.device);
    for (uint32_t m : p.mask) p.unsupported += (uint64_t)__builtin_popcount(m);
}

// A locus of one contig: its first unsupported window a, and whether its candidates are tried.
struct Locus { uint64_t a; bool attempted; };

// Contig c's loci in ascending a: the maximal runs of consecutive unsupported window starts (on a circular contig a run may wrap), each
// attempted when window a-1 exists and is supported (and a circular contig is at least 2k + 2L long).
std::vector<Locus> loci_of(const Packed& p, size_t c, uint64_t n, bool circular, uint32_t k, uint32_t L) {
    std::vector<std::pair<uint64_t, uint64_t>> runs;
    for (uint64_t j = p.woff[c]; j < p.woff[c + 1]; ++j)
        for (uint32_t bits = p.mask[j]; bits; bits &= bits - 1) {
            const uint64_t s = 32 * (j - p.woff[c]) + (uint64_t)__builtin_ctz(bits) + 1 - k;
            if (!runs.empty() && runs.back().second + 1 == s) runs.back().second = s;
            else runs.emplace_back(s, s);
        }
    const bool whole = circular && runs.size() == 1 && runs[0].first == 0 && runs[0].second == n - 1;
    if (circular && runs.size() > 1 && runs.front().first == 0 && runs.back().second == n - 1) {
        runs.front().first = runs.back().first;              // the run that wraps starts at the last run's start
        runs.pop_back();
    }
    const char* b = p.bytes.data() + p.off[c];
    auto valid = [&](uint64_t j) { for (uint32_t i = 0; i < k; ++i) if (!acgt(b[j + i])) return false; return true; };
    std::vector<Locus> out;
    for (const auto& run : runs) {
        const uint64_t a = run.first;
        bool attempted;
        if (circular) attempted = !whole && n >= 2ull * k + 2ull * L && valid(a ? a - 1 : n - 1);
        else attempted = a >= 1 && valid(a - 1);
        out.push_back(Locus{a, attempted});
    }
    std::sort(out.begin(), out.end(), [](const Locus& x, const Locus& y) { return x.a < y.a; });
    return out;
}
}  // namespace

void polish_run(DeviceSubsample& sub, DeviceSpectrum& spec, DevicePolish& dev, const std::string& assembly, const std::string& reads, uint32_t k,
                const uint32_t* min_count, uint32_t L, uint32_t max_rounds, uint64_t window, PolishResult& out) {
    out = PolishResult();
    out.recs = load_fasta(assembly);
    std::vector<FastaRecord>& recs = out.recs;
    if (recs.size() >= 0xFFFFFFFFull) throw RangeError{"polish: 2^32 - 1 contigs or more"};
    // the buffers every round can need: each kept edit's span holds at least 2k - 1 bases and adds at most L of them
    uint64_t bytes = 0, windows = 0;
    {
        std::string b;
        for (const FastaRecord& r : recs) windows += pack_contig(r, k, b);
        bytes = b.size();
    }
    if (!windows) throw InputError{assembly + ": no k-mer windows: no contig holds " + std::to_string(k) + " consecutive A, C, G or T bases"};
    const uint64_t n_contigs = recs.size();
    for (uint32_t r = 0; r < max_rounds; ++r) bytes += L * (bytes / (2 * k - 1) + n_contigs);
    bytes += (k - 1) * n_contigs;                                  // a circular contig that grows to k bases gains its junction
    const uint64_t budget_env = genome_size_env("AC_POLISH_TABLE_SLOTS");
    dev.reserve(bytes, bytes / 32 + n_contigs, bytes, k, budget_env ? budget_env : ac_gs_budget_slots(), &out.device);
    const ReadPass pass = pack_reads(sub, spec, reads, k, window);
    out.reads = pass.reads; out.read_ms = pass.read_ms; out.copy_ms = pass.copy_ms;
    spec.totals(&out.read_windows, &out.read_bases);
    if (!out.read_windows) throw InputError{"no k-mer windows: no read holds " + std::to_string(k) + " consecutive A, C, G or T bases"};
    std::vector<uint64_t> hist(AC_GS_BINS, 0);
    const uint64_t budget = genome_size_env("AC_GS_TABLE_SLOTS");         // read after the window table exists: half of what is left
    spec.count(out.read_windows, budget ? budget : ac_gs_budget_slots(), genome_size_env("AC_GS_PARTITIONS"), hist.data(), &out.spectrum);
    for (uint64_t c = 1; c < AC_GS_BINS; ++c) out.distinct += hist[c];
    out.valley = genome_size_valley(hist.data());
    if (!min_count && !out.valley)
        throw InputError{std::string(genome_size_no_peak) + "; --min_count sets the solid threshold without it"};
    const uint32_t t = min_count ? *min_count : (uint32_t)out.valley;
    out.min_count = t;

    Packed p;
    evaluate(dev, spec, recs, k, t, p, out);
    out.kmers_before = p.windows; out.unsupported_before = p.unsupported;
    for (uint32_t round = 1; round <= max_rounds; ++round) {
        auto t0 = std::chrono::steady_clock::now();
        PolishRound rd;
        rd.unsupported = p.unsupported;
        std::vector<std::vector<Locus>> loci(recs.size());
        std::vector<PlLocus> tried;
        for (size_t c = 0; c < recs.size(); ++c) {
            const uint64_t n = recs[c].seq.size();
            const bool circular = p.len[c] > n;
            loci[c] = loci_of(p, c, n, circular, k, L);
            rd.loci += loci[c].size();
            for (const Locus& l : loci[c])
                if (l.attempted) tried.push_back(PlLocus{p.woff[c], n, l.a, circular ? 1u : 0u, 0});
                else ++rd.edge;
        }
        out.host_ms += ms_since(t0);
        std::vector<uint32_t> choice(3 * tried.size());
        dev.choose(spec, tried.data(), tried.size(), L, t, budget_env ? budget_env : ac_gs_budget_slots(), choice.data(), &out.device);
        t0 = std::chrono::steady_clock::now();
        // per contig: the accepted edits in ascending a, kept unless their span overlaps a kept one's, then applied in one pass
        struct Kept { uint64_t p0; PlEdit e; uint32_t score; };
        size_t next = 0;
        for (size_t c = 0; c < recs.size(); ++c) {
            std::string& s = recs[c].seq;
            const uint64_t n = s.size();
            const bool circular = p.len[c] > n;
            std::vector<Kept> kept;
            uint64_t max_end = 0, first_a = 0;
            for (const Locus& l : loci[c]) {
                if (!l.attempted) continue;
                const uint32_t* o = choice.data() + 3 * next++;
                if (!o[0]) { ++rd.none; continue; }
                if (o[1] > 1) { ++rd.ambiguous; continue; }
                const uint64_t p0 = (l.a + k - 1) % n;
                const PlEdit e = pl_edit(o[2], L, code_of(s[p0]));
                const uint64_t d = e.mlen ? 0 : e.skip, end = l.a + 2 * k - 1 + d;
                if (!kept.empty() && (l.a < max_end || (circular && end > n && end - n > first_a))) { ++rd.deferred; continue; }
                if (kept.empty()) first_a = l.a;
                max_end = std::max(max_end, end);
                kept.push_back(Kept{p0, e, o[0]});
            }
            std::sort(kept.begin(), kept.end(), [](const Kept& x, const Kept& y) { return x.p0 < y.p0; });
            std::string polished;
            uint64_t at = 0;
            for (const Kept& e : kept) {
                std::string mid;
                for (uint32_t i = 0; i < e.e.mlen; ++i) mid += BASES[(e.e.mid >> (2 * i)) & 3];
                const std::string ref = e.e.skip ? s.substr(e.p0, e.e.skip) : "-";
                out.edits_tsv += std::to_string(round) + "\t" + recs[c].name + "\t" + std::to_string(e.p0) + "\t" + ref + "\t" +
                                 (mid.empty() ? "-" : mid) + "\t" + std::to_string(e.score) + "\n";
                polished.append(s, at, e.p0 - at);
                polished += mid;
                at = e.p0 + e.e.skip;
            }
            if (!kept.empty()) s = polished.append(s, at, std::string::npos);
            rd.edited += kept.size();
        }
        if (next != tried.size()) throw std::logic_error("polish: the choices are not the tried loci");
        out.edits += rd.edited;
        out.rounds.push_back(rd);
        out.host_ms += ms_since(t0);
        if (!rd.edited) break;
        evaluate(dev, spec, recs, k, t, p, out);
    }
    out.kmers_after = p.windows; out.unsupported_after = p.unsupported;
    const auto t0 = std::chrono::steady_clock::now();
    for (size_t c = 0; c < recs.size(); ++c)
        contig_bed(recs[c].name, recs[c].seq.size(), p.mask.data() + p.woff[c], p.woff[c + 1] - p.woff[c], k, out.bed);
    out.host_ms += ms_since(t0);
    out.scan_ms = sub.kernel_ms;
    out.pack_reads_ms = spec.packed_ms();
    out.kernel_ms = sub.kernel_ms + spec.kernel_ms + out.device.pack_ms + out.device.fill_ms + out.device.sweep.count_ms + out.device.candidate_ms +
                    out.device.choose_ms;
}

std::string polish_fasta(const PolishResult& r) {
    std::string t;
    for (const FastaRecord& rec : r.recs) t += ">" + rec.header + "\n" + rec.seq + "\n";
    return t;
}

std::string polish_edits(const PolishResult& r) { return "round\tcontig\tposition\tref\talt\tscore\n" + r.edits_tsv; }

std::string polish_rounds(const PolishResult& r) {
    std::string t = "round\tunsupported\tloci\tedited\tambiguous\tnone\tedge\tdeferred\n";
    for (size_t i = 0; i < r.rounds.size(); ++i) {
        const PolishRound& x = r.rounds[i];
        t += std::to_string(i + 1) + "\t" + std::to_string(x.unsupported) + "\t" + std::to_string(x.loci) + "\t" + std::to_string(x.edited) + "\t" +
             std::to_string(x.ambiguous) + "\t" + std::to_string(x.none) + "\t" + std::to_string(x.edge) + "\t" + std::to_string(x.deferred) + "\n";
    }
    return t;
}

std::string polish_summary(const PolishResult& r, uint32_t k) {
    return "contigs\tkmers_before\tunsupported_before\tqv_before\tedits\tkmers_after\tunsupported_after\tqv_after\tmin_count\trounds\n" +
           std::to_string(r.recs.size()) + "\t" + std::to_string(r.kmers_before) + "\t" + std::to_string(r.unsupported_before) + "\t" +
           qv_text(r.unsupported_before, r.kmers_before, k) + "\t" + std::to_string(r.edits) + "\t" + std::to_string(r.kmers_after) + "\t" +
           std::to_string(r.unsupported_after) + "\t" + qv_text(r.unsupported_after, r.kmers_after, k) + "\t" + std::to_string(r.min_count) + "\t" +
           std::to_string(r.rounds.size()) + "\n";
}
