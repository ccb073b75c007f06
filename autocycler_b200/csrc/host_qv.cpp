// `autocycler qv` on the host (see host_qv.h and DESIGN.md §20).
#include "host_qv.h"

#include <sys/stat.h>

#include <algorithm>
#include <cmath>
#include <cstdio>

#include "host_depth.h"
#include "host_genome_size.h"
#include "host_subsample.h"

std::vector<std::string> qv_inputs(const std::vector<std::string>& args) {
    std::vector<std::string> out;
    for (const std::string& a : args) {
        struct stat st;
        if (stat(a.c_str(), &st) != 0) throw InputError{"file does not exist: " + a};
        if (S_ISDIR(st.st_mode)) {
            const std::vector<std::string> found = find_all_assemblies(a);
            out.insert(out.end(), found.begin(), found.end());
        } else {
            out.push_back(a);
        }
    }
    return out;
}

std::string qv_text(uint64_t unsupported, uint64_t kmers, uint32_t k) {
    if (!kmers) return "";
    if (!unsupported) return "inf";
    const double p = -std::expm1(std::log1p(-(double)unsupported / (double)kmers) / (double)k);
    char buf[64];
    snprintf(buf, sizeof buf, "%.2f", -10.0 * std::log10(p) + 0.0);          // + 0.0: E = K gives 0.00, not -0.00
    return buf;
}

namespace {
std::string percent(uint64_t num, uint64_t den) {
    if (!den) return "";
    char buf[64];
    snprintf(buf, sizeof buf, "%.2f", 100.0 * (double)num / (double)den);
    return buf;
}

}  // namespace

void contig_bed(const std::string& name, uint64_t L, const uint32_t* mask, uint64_t words, uint32_t k, std::string& bed) {
    std::vector<std::pair<uint64_t, uint64_t>> iv;
    for (uint64_t j = 0; j < words; ++j)
        for (uint32_t bits = mask[j]; bits; bits &= bits - 1) {
            const uint64_t p = 32 * j + (uint64_t)__builtin_ctz(bits) + 1 - k;
            if (p + k <= L) { iv.emplace_back(p, p + k); continue; }
            iv.emplace_back(p, L);
            iv.emplace_back(0, p + k - L);
        }
    std::sort(iv.begin(), iv.end());
    for (size_t i = 0; i < iv.size();) {
        uint64_t s = iv[i].first, e = iv[i].second;
        for (++i; i < iv.size() && iv[i].first <= e; ++i) e = std::max(e, iv[i].second);
        bed += name + "\t" + std::to_string(s) + "\t" + std::to_string(e) + "\n";
    }
}

void qv_run(DeviceSubsample& sub, DeviceSpectrum& spec, DeviceQv& dev, const std::vector<std::string>& paths, const std::string& reads,
            uint32_t k, const uint32_t* min_count, uint64_t window, QvResult& out) {
    out = QvResult();
    // every assembly's contigs back to back, as depth packs one assembly's
    std::string bytes;
    std::vector<uint64_t> len, windows;
    std::vector<uint32_t> first{0};
    for (const std::string& path : paths) {
        const std::vector<FastaRecord> recs = load_fasta(path);
        QvAssembly as;
        as.path = path;
        uint64_t aw = 0;
        for (const FastaRecord& r : recs) {
            const size_t start = bytes.size();
            QvContig c;
            c.name = r.name; c.length = r.seq.size(); c.kmers = pack_contig(r, k, bytes);
            len.push_back(bytes.size() - start);
            aw += c.kmers;
            as.contigs.push_back(std::move(c));
        }
        if (!aw) throw InputError{path + ": no k-mer windows: no contig holds " + std::to_string(k) + " consecutive A, C, G or T bases"};
        if (len.size() >= 0xFFFFFFFFull) throw RangeError{"qv: 2^32 - 1 contigs or more"};
        as.kmers = aw;
        windows.push_back(aw);
        first.push_back((uint32_t)len.size());
        out.assemblies.push_back(std::move(as));
    }
    const uint32_t n_asm = (uint32_t)out.assemblies.size();
    const uint64_t budget_env = genome_size_env("AC_QV_TABLE_SLOTS");
    dev.build((const uint8_t*)bytes.data(), len.data(), (uint32_t)len.size(), first.data(), n_asm, windows.data(), k,
              budget_env ? budget_env : ac_gs_budget_slots(), &out.device);
    const ReadPass pass = pack_reads(sub, spec, reads, k, window);
    out.reads = pass.reads; out.read_ms = pass.read_ms; out.copy_ms = pass.copy_ms;
    spec.totals(&out.read_windows, &out.read_bases);
    if (!out.read_windows) throw InputError{"no k-mer windows: no read holds " + std::to_string(k) + " consecutive A, C, G or T bases"};
    dev.probe(spec, &out.device);
    out.hist.assign(AC_GS_BINS, 0);
    const uint64_t budget = genome_size_env("AC_GS_TABLE_SLOTS");          // read after the qv tables exist: half of what is left
    spec.count(out.read_windows, budget ? budget : ac_gs_budget_slots(), genome_size_env("AC_GS_PARTITIONS"), out.hist.data(), &out.spectrum);
    const uint64_t* h = out.hist.data();
    for (uint64_t c = 1; c < AC_GS_BINS; ++c) out.distinct += h[c];
    out.valley = genome_size_valley(h);
    if (!min_count && !out.valley)
        throw InputError{std::string(genome_size_no_peak) + "; --min_count sets the solid threshold without it"};
    const uint64_t t = min_count ? *min_count : out.valley;
    out.min_count = t;
    for (uint64_t c = t; c < AC_GS_BINS; ++c) out.solid += h[c];
    const std::vector<uint64_t>& woff = dev.word_offsets();
    std::vector<uint32_t> mask, cn((size_t)AC_GS_BINS * AC_QV_CN);
    for (uint32_t a = 0; a < n_asm; ++a) {
        QvAssembly& as = out.assemblies[a];
        mask.resize(woff[first[a + 1]] - woff[first[a]]);
        dev.assembly(a, (uint32_t)t, mask.data(), cn.data(), &out.device);
        for (uint32_t i = 0; i < as.contigs.size(); ++i) {
            QvContig& c = as.contigs[i];
            const uint64_t g = first[a] + i, at = woff[g] - woff[first[a]], words = woff[g + 1] - woff[g];
            for (uint64_t j = 0; j < words; ++j) c.unsupported += (uint64_t)__builtin_popcount(mask[at + j]);
            as.unsupported += c.unsupported;
            contig_bed(c.name, c.length, mask.data() + at, words, k, as.bed);
        }
        as.spectrum = "count\tcn0\tcn1\tcn2\tcn3\tcn4+\n";
        for (uint64_t c = 0; c < AC_GS_BINS; ++c) {
            const uint32_t* row = cn.data() + c * AC_QV_CN;
            uint64_t in_asm = 0;
            for (uint32_t m = 1; m < AC_QV_CN; ++m) in_asm += row[m];
            if (c >= t) as.solid_found += in_asm;
            if (c && in_asm > h[c]) throw std::logic_error("qv: an assembly holds more keys in a bin than the reads");
            const uint64_t cn0 = c ? h[c] - in_asm : 0;
            if (!cn0 && !in_asm) continue;
            as.spectrum += std::to_string(c) + "\t" + std::to_string(cn0);
            for (uint32_t m = 1; m < AC_QV_CN; ++m) as.spectrum += "\t" + std::to_string(row[m]);
            as.spectrum += "\n";
        }
    }
    out.scan_ms = sub.kernel_ms;
    out.pack_reads_ms = spec.packed_ms();
    out.kernel_ms = sub.kernel_ms + spec.kernel_ms + out.device.pack_ms + out.device.insert_ms + out.device.probe_ms + out.device.assembly_ms;
}

std::string qv_table(const QvResult& r, uint32_t k) {
    std::string t = "assembly\tkmers\tunsupported\tqv\tsolid_found\tsolid_kmers\tcompleteness\tmin_count\n";
    for (const QvAssembly& a : r.assemblies)
        t += a.path + "\t" + std::to_string(a.kmers) + "\t" + std::to_string(a.unsupported) + "\t" + qv_text(a.unsupported, a.kmers, k) + "\t" +
             std::to_string(a.solid_found) + "\t" + std::to_string(r.solid) + "\t" + percent(a.solid_found, r.solid) + "\t" +
             std::to_string(r.min_count) + "\n";
    return t;
}

std::string qv_contig_table(const QvResult& r, uint32_t k) {
    std::string t = "assembly\tcontig\tlength\tkmers\tunsupported\tqv\n";
    for (const QvAssembly& a : r.assemblies)
        for (const QvContig& c : a.contigs)
            t += a.path + "\t" + c.name + "\t" + std::to_string(c.length) + "\t" + std::to_string(c.kmers) + "\t" + std::to_string(c.unsupported) +
                 "\t" + qv_text(c.unsupported, c.kmers, k) + "\n";
    return t;
}

std::string qv_histogram(const QvResult& r) {
    std::string t;
    for (uint64_t c = 1; c < AC_GS_BINS; ++c)
        if (r.hist[c]) t += std::to_string(c) + "\t" + std::to_string(r.hist[c]) + "\n";
    return t;
}
