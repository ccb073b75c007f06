// `autocycler depth` on the host (see host_depth.h and DESIGN.md §19).  Citations are file:line in the reference's src/.
#include "host_depth.h"

#include <algorithm>
#include <cmath>
#include <cstdio>

#include "host_genome_size.h"
#include "host_subsample.h"

bool depth_from_header(const std::string& header, double& depth) {
    size_t at = header.find("depth=");
    size_t from = at + 6;
    if (at == std::string::npos) { at = header.find("depth-"); from = at + 6; }
    if (at == std::string::npos) { at = header.find("coverage="); from = at + 9; }
    if (at == std::string::npos) return false;
    std::string num = header.substr(from, header.find_first_of("-_ ", from) - from);   // split(['-', '_', ' ']).next()
    for (char& c : num) if (c >= 'A' && c <= 'Z') c = (char)(c + 32);                  // Rust's f64 grammar is case-insensitive
    return rust_f64(num, depth);
}

std::string rust_fixed(double x, int digits) {
    if (std::isnan(x)) return "NaN";
    if (std::isinf(x)) return x > 0 ? "inf" : "-inf";
    char buf[512];
    snprintf(buf, sizeof buf, "%.*f", digits, x);                   // both round the exact binary value to nearest, ties to even
    return buf;
}

bool depth_filter(const std::vector<FastaRecord>& recs, const std::vector<double>& depth, const std::vector<char>& has, const double* min_abs,
                  const double* min_rel, std::vector<char>& keep, std::string& report) {
    keep.assign(recs.size(), 1);
    if (!min_abs && !min_rel) return false;
    size_t longest_len = 0;
    double longest_depth = 0.0;
    for (size_t i = 0; i < recs.size(); ++i) {
        if (!has[i]) return false;
        if (recs[i].seq.size() > longest_len) { longest_len = recs[i].seq.size(); longest_depth = depth[i]; }
    }
    double threshold = min_abs ? *min_abs : 0.0;
    if (min_rel) threshold = std::fmax(threshold, *min_rel * longest_depth);    // f64::max: a NaN side gives the other
    report += "\nAutocycler helper depth filter\nthreshold = " + rust_fixed(threshold, 3) + "\n";
    for (size_t i = 0; i < recs.size(); ++i) {
        keep[i] = depth[i] >= threshold;
        report += recs[i].name + ": depth=" + rust_fixed(depth[i], 3) + ", " + (keep[i] ? "PASS" : "FAIL") + "\n";
    }
    return true;
}

std::string depth_filter_text(const std::string& text, const std::string& name, const double* min_abs, const double* min_rel,
                              std::string& report) {
    if (!min_abs && !min_rel) return text;
    std::vector<FastaRecord> recs = parse_fasta(text, name);
    size_t bases = 0;
    for (const FastaRecord& r : recs) bases += r.seq.size();
    if (bases == 0) return text;                                          // is_fasta_empty
    check_fasta(recs, name);
    std::vector<double> depth(recs.size());
    std::vector<char> has(recs.size()), keep;
    for (size_t i = 0; i < recs.size(); ++i) has[i] = depth_from_header(recs[i].header, depth[i]);
    if (!depth_filter(recs, depth, has, min_abs, min_rel, keep, report)) return text;
    std::string out;
    for (size_t i = 0; i < recs.size(); ++i)
        if (keep[i]) out += ">" + recs[i].header + "\n" + recs[i].seq + "\n";
    return out;
}

uint64_t pack_contig(const FastaRecord& r, uint32_t k, std::string& bytes) {
    std::string lower = r.header;
    for (char& ch : lower) if (ch >= 'A' && ch <= 'Z') ch = (char)(ch + 32);
    const bool circular = lower.find("circular=true") != std::string::npos && r.seq.size() >= k;    // rotate_plassembler_contigs' test, helper.rs:866
    const size_t start = bytes.size();
    bytes += r.seq;
    if (circular) bytes.append(r.seq, 0, k - 1);
    uint64_t run = 0, windows = 0;
    for (size_t i = start; i < bytes.size(); ++i) {
        const char b = bytes[i];
        run = (b == 'A' || b == 'C' || b == 'G' || b == 'T') ? run + 1 : 0;
        windows += run >= k;
    }
    return windows;
}

void depth_run(DeviceSubsample& sub, DeviceSpectrum& spec, DeviceDepth& dev, const std::string& assembly, const std::string& reads, uint32_t k,
               uint64_t window, DepthResult& out) {
    out = DepthResult();
    out.recs = load_fasta(assembly);
    const std::vector<FastaRecord>& recs = out.recs;
    for (const FastaRecord& r : recs) {
        double d;
        if (depth_from_header(r.header, d))
            throw InputError{assembly + ": the header of " + r.name + " already carries a depth; use --source header to filter by it"};
    }
    std::string bytes;
    std::vector<uint64_t> len(recs.size());
    uint64_t windows = 0;
    for (size_t c = 0; c < recs.size(); ++c) {
        const size_t start = bytes.size();
        windows += pack_contig(recs[c], k, bytes);
        len[c] = bytes.size() - start;
    }
    const uint64_t budget_env = genome_size_env("AC_DEPTH_TABLE_SLOTS");
    const uint64_t budget = budget_env ? budget_env : ac_gs_budget_slots();
    dev.build((const uint8_t*)bytes.data(), len.data(), (uint32_t)std::min<size_t>(recs.size(), 0xFFFFFFFFu), windows, k, budget, &out.device);
    const ReadPass pass = pack_reads(sub, spec, reads, k, window);
    out.reads = pass.reads; out.read_ms = pass.read_ms; out.copy_ms = pass.copy_ms;
    spec.totals(&out.read_windows, &out.read_bases);
    dev.probe(spec, &out.device);
    out.unique.assign(recs.size(), 0);
    out.depth.assign(recs.size(), NAN);
    dev.medians(out.unique.data(), out.depth.data(), &out.device);
    for (uint64_t u : out.unique) out.unique_total += u;
    out.scan_ms = sub.kernel_ms;
    out.pack_reads_ms = spec.packed_ms();
    out.kernel_ms = sub.kernel_ms + out.pack_reads_ms + out.device.pack_ms + out.device.insert_ms + out.device.probe_ms + out.device.median_ms;
}
