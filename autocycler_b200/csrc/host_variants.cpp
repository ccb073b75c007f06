// `autocycler variants` on the host (see host_variants.h and DESIGN.md §23).
#include "host_variants.h"

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <stdexcept>

#include "host_depth.h"
#include "host_genome_size.h"
#include "host_subsample.h"

namespace {
double ms_since(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

// 0..3 for A, C, G, T in either case, else -1.
int code_of(char b) {
    switch (b) {
        case 'A': case 'a': return 0;
        case 'C': case 'c': return 1;
        case 'G': case 'g': return 2;
        case 'T': case 't': return 3;
        default: return -1;
    }
}
const char* const BASES = "ACGT";

// The polish object's std::length_error, in this command's words.
[[noreturn]] void rethrow_as_variants(const std::length_error& e) {
    std::string m = e.what();
    if (m.rfind("polish:", 0) == 0) m = "variants:" + m.substr(7);
    throw std::length_error(m);
}

// A candidate to measure: its locus (one per position with any), contig, position p and index in pl_edit's order.
struct Want { uint64_t locus; uint32_t contig, c; uint64_t p; };

// The row of candidate c evaluated at p of the uppercased sequence s, an indel shifted left while p > 1 and the base before it equals the
// event's last base, then anchored on the base before it (POS = p), or on the base after it at POS 1 when it sits at p = 0.
VariantRow vcf_row(const std::string& s, uint64_t p, uint32_t c, uint32_t L) {
    const PlEdit e = pl_edit(c, L, (uint32_t)code_of(s[p]));
    VariantRow row;
    row.p = p; row.c = c;
    if (c < 3) {
        row.pos = p + 1; row.ref_allele = s.substr(p, 1); row.alt_allele = std::string(1, BASES[e.mid]);
    } else if (!e.mlen) {
        const uint64_t d = e.skip;
        while (p > 1 && s[p - 1] == s[p + d - 1]) --p;
        if (p == 0) { row.pos = 1; row.ref_allele = s.substr(0, d + 1); row.alt_allele = s.substr(d, 1); }
        else { row.pos = p; row.ref_allele = s.substr(p - 1, d + 1); row.alt_allele = s.substr(p - 1, 1); }
    } else {
        std::string ins;
        for (uint32_t i = 0; i < e.mlen; ++i) ins += BASES[(e.mid >> (2 * i)) & 3];
        while (p > 1 && s[p - 1] == ins.back()) { ins = ins.back() + ins.substr(0, ins.size() - 1); --p; }
        if (p == 0) { row.pos = 1; row.ref_allele = s.substr(0, 1); row.alt_allele = ins + s[0]; }
        else { row.pos = p; row.ref_allele = s.substr(p - 1, 1); row.alt_allele = s[p - 1] + ins; }
    }
    return row;
}
}  // namespace

void variants_run(DeviceSubsample& sub, DeviceSpectrum& spec, DevicePolish& pl, DeviceVariants& dev, const std::string& assembly,
                  const std::string& reads, uint32_t k, const uint32_t* min_count, uint32_t L, double min_fraction, uint64_t window,
                  VariantsResult& out) {
    out = VariantsResult();
    out.recs = load_fasta(assembly);
    const std::vector<FastaRecord>& recs = out.recs;
    if (recs.size() >= 0xFFFFFFFFull) throw RangeError{"variants: 2^32 - 1 contigs or more"};
    auto t0 = std::chrono::steady_clock::now();
    std::string bytes;
    std::vector<uint64_t> off, len, woff{0};                    // per contig: first byte, bytes (junction bases included), first packed word
    for (const FastaRecord& r : recs) {
        off.push_back(bytes.size());
        out.kmers += pack_contig(r, k, bytes);
        len.push_back(bytes.size() - off.back());
        woff.push_back(woff.back() + len.back() / 32 + 1);
    }
    if (!out.kmers) throw InputError{assembly + ": no k-mer windows: no contig holds " + std::to_string(k) + " consecutive A, C, G or T bases"};
    out.host_ms += ms_since(t0);
    const uint64_t budget_env = genome_size_env("AC_VARIANTS_TABLE_SLOTS");
    try {
        pl.reserve(std::max<uint64_t>(bytes.size(), 1), woff.back(), out.kmers, k, budget_env ? budget_env : ac_gs_budget_slots(), &out.device);
    } catch (const std::length_error& e) { rethrow_as_variants(e); }
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

    pl.pack((const uint8_t*)bytes.data(), len.data(), (uint32_t)recs.size(), out.kmers, &out.device);
    std::vector<uint32_t> mask(3 * woff.back());
    dev.screen(spec, pl, t, mask.data(), &out.device, &out.va);

    // the tried positions, the screened ones, and the rightmost candidates whose first window S(p, e) passes the screen
    t0 = std::chrono::steady_clock::now();
    const uint32_t C = (uint32_t)DevicePolish::candidates(L);
    std::vector<std::string> up(recs.size());
    std::vector<PlLocus> loci;
    std::vector<Want> want;
    for (size_t c = 0; c < recs.size(); ++c) {
        std::string& s = up[c];
        s = recs[c].seq;
        for (char& ch : s) if (ch >= 'a' && ch <= 'z') ch = (char)(ch - 32);
        const uint64_t n = s.size();
        const bool circular = len[c] > n;
        const char* ext = bytes.data() + off[c];
        std::vector<uint32_t> run(len[c]);                    // A/C/G/T bases that end at each packed byte
        for (uint64_t i = 0; i < len[c]; ++i) run[i] = code_of(ext[i]) >= 0 ? (i ? run[i - 1] : 0) + 1 : 0;
        const uint64_t first = circular ? (n >= 2ull * k + 2ull * L ? 0 : n) : k - 1;
        for (uint64_t p = first; p < n; ++p) {
            const uint64_t idx = circular && p < k - 1 ? n + p : p;       // the packed base the window ending at p ends at
            if (run[idx] < k) continue;
            ++out.positions;
            const uint64_t w = woff[c] + idx / 32;
            const uint32_t o = (uint32_t)(idx % 32);
            const uint32_t bits = ((mask[3 * w] >> o) & 1u) | (((mask[3 * w + 1] >> o) & 1u) << 1) | (((mask[3 * w + 2] >> o) & 1u) << 2);
            if (!bits) continue;
            ++out.screened;
            const int cur = code_of(s[p]);
            bool any = false;
            for (uint32_t x = 0; x < C; ++x) {
                const PlEdit e = pl_edit(x, L, (uint32_t)cur);
                int b;
                if (e.mlen) b = (int)(e.mid & 3u);
                else {
                    if (p + e.skip >= n + (circular ? 1 : 0)) continue;
                    b = code_of(s[(p + e.skip) % n]);
                }
                if (b < 0 || b == cur || !((bits >> (b < cur ? b : b - 1)) & 1u)) continue;
                ++out.candidates;
                if (!any) loci.push_back(PlLocus{woff[c], n, circular ? (p + n - (k - 1)) % n : p - (k - 1), circular ? 1u : 0u, 0});
                any = true;
                want.push_back(Want{loci.size() - 1, (uint32_t)c, x, p});
            }
        }
    }
    out.loci = loci.size();
    out.host_ms += ms_since(t0);
    std::vector<uint32_t> score(loci.size() * C);
    try {
        dev.scores(spec, pl, loci.data(), loci.size(), L, t, budget_env ? budget_env : ac_gs_budget_slots(), score.data(), &out.device);
    } catch (const std::length_error& e) { rethrow_as_variants(e); }
    std::vector<VaCandidate> passing;
    std::vector<const Want*> passing_want;
    for (const Want& x : want)
        if (score[x.locus * C + x.c]) { passing.push_back(VaCandidate{loci[x.locus], x.c, 0}); passing_want.push_back(&x); }
    out.passing = passing.size();
    std::vector<uint32_t> rk(2 * passing.size());
    dev.ref(pl, passing.data(), passing.size(), L, rk.data(), &out.va);

    t0 = std::chrono::steady_clock::now();
    for (size_t i = 0; i < passing.size(); ++i) {
        const Want& x = *passing_want[i];
        const uint32_t alt = score[x.locus * C + x.c], ref = rk[2 * i], pk = rk[2 * i + 1];
        if (!((double)alt >= min_fraction * ((double)alt + (double)ref))) continue;
        VariantRow row = vcf_row(up[x.contig], x.p, x.c, L);
        row.contig = x.contig; row.alt = alt; row.ref = ref; row.pk = pk;
        if (x.c < 3) ++out.substitutions;
        else if (row.ref_allele.size() > row.alt_allele.size()) ++out.deletions;
        else ++out.insertions;
        out.paralog += pk > 0; out.alt_major += alt > ref;
        out.rows.push_back(std::move(row));
    }
    std::sort(out.rows.begin(), out.rows.end(), [](const VariantRow& a, const VariantRow& b) {
        if (a.contig != b.contig) return a.contig < b.contig;
        if (a.pos != b.pos) return a.pos < b.pos;
        if (a.p != b.p) return a.p < b.p;
        return a.c < b.c;
    });
    out.host_ms += ms_since(t0);
    out.scan_ms = sub.kernel_ms;
    out.pack_reads_ms = spec.packed_ms();
    out.kernel_ms = sub.kernel_ms + spec.kernel_ms + out.device.pack_ms + out.device.fill_ms + out.device.sweep.count_ms + out.device.candidate_ms +
                    out.va.screen_ms + out.va.ref_ms;
}

std::string variants_vcf(const VariantsResult& r) {
    std::string t = "##fileformat=VCFv4.2\n##source=autocycler variants\n";
    for (const FastaRecord& rec : r.recs) t += "##contig=<ID=" + rec.name + ",length=" + std::to_string(rec.seq.size()) + ">\n";
    t += "##INFO=<ID=AF,Number=A,Type=Float,Description=\"Alternative allele fraction AK / (AK + RK)\">\n"
         "##INFO=<ID=AK,Number=A,Type=Integer,Description=\"Least read count of the k-mers that carry the alternative allele\">\n"
         "##INFO=<ID=RK,Number=1,Type=Integer,Description=\"Least read count of the assembly k-mers the alternative allele replaces\">\n"
         "##INFO=<ID=PK,Number=A,Type=Integer,Description=\"Alternative-allele k-mers that occur elsewhere in the assembly\">\n"
         "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n";
    char af[32];
    for (const VariantRow& x : r.rows) {
        snprintf(af, sizeof af, "%.4f", (double)x.alt / ((double)x.alt + (double)x.ref));
        t += r.recs[x.contig].name + "\t" + std::to_string(x.pos) + "\t.\t" + x.ref_allele + "\t" + x.alt_allele + "\t.\tPASS\tAF=" + af +
             ";AK=" + std::to_string(x.alt) + ";RK=" + std::to_string(x.ref) + ";PK=" + std::to_string(x.pk) + "\n";
    }
    return t;
}

std::string variants_summary(const VariantsResult& r) {
    return "contigs\tpositions\tscreened\tcandidates\tvariants\tsubstitutions\tinsertions\tdeletions\tparalog\talt_major\tmin_count\n" +
           std::to_string(r.recs.size()) + "\t" + std::to_string(r.positions) + "\t" + std::to_string(r.screened) + "\t" +
           std::to_string(r.candidates) + "\t" + std::to_string(r.rows.size()) + "\t" + std::to_string(r.substitutions) + "\t" +
           std::to_string(r.insertions) + "\t" + std::to_string(r.deletions) + "\t" + std::to_string(r.paralog) + "\t" +
           std::to_string(r.alt_major) + "\t" + std::to_string(r.min_count) + "\n";
}
