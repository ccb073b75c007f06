// Stage A of compress on the host (see host_io.h).  Citations are file:line in the reference's src/.
#include "host_io.h"

#include <dirent.h>
#include <sys/stat.h>
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstring>
#include <thread>
#include <unordered_map>
#include <unordered_set>

static void fail(const std::string& m) { throw InputError{m}; }

static bool has_suffix(const std::string& s, const char* suf) {
    size_t n = strlen(suf); return s.size() >= n && memcmp(s.data() + s.size() - n, suf, n) == 0;
}

// misc.rs:86-95.  `&&` binds tighter than `||` in the reference's expression, so a file whose stem ends in
// ".fna" or ".fa" qualifies whatever its extension is (e.g. "x.fa.bak"); only ".fasta" stems need ".gz".
static bool is_assembly_file(const std::string& dir, const std::string& name) {
    struct stat st;
    if (stat((dir + "/" + name).c_str(), &st) != 0 || !S_ISREG(st.st_mode)) return false;
    size_t dot = name.rfind('.');
    std::string stem = name, ext;
    if (dot != std::string::npos && dot != 0) { stem = name.substr(0, dot); ext = name.substr(dot + 1); }
    if (ext == "fasta" || ext == "fna" || ext == "fa") return true;
    if (ext == "gz" && has_suffix(stem, ".fasta")) return true;
    return has_suffix(stem, ".fna") || has_suffix(stem, ".fa");
}

std::vector<std::string> find_all_assemblies(const std::string& dir_in) {   // misc.rs:64-83
    std::string dir = dir_in;
    while (dir.size() > 1 && dir.back() == '/') dir.pop_back();
    DIR* d = opendir(dir.c_str());
    if (!d) fail("unable to read directory " + dir_in);
    std::vector<std::string> found;
    for (dirent* e; (e = readdir(d)) != nullptr;) {
        std::string name = e->d_name;
        if (name == "." || name == "..") continue;
        if (is_assembly_file(dir, name)) found.push_back(dir + "/" + name);
    }
    closedir(d);
    std::sort(found.begin(), found.end());
    if (found.empty()) fail("no assemblies found in " + dir_in);
    return found;
}

static std::string slurp(const std::string& path) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) fail("unable to load " + path);
    unsigned char magic[2] = {0, 0};
    size_t got = fread(magic, 1, 2, f);
    std::string data;
    if (got == 2 && magic[0] == 0x1f && magic[1] == 0x8b) {   // misc.rs:233-245 gzip magic; flate2 MultiGzDecoder
        fclose(f);
        gzFile g = gzopen(path.c_str(), "rb");
        if (!g) fail("unable to load " + path);
        std::vector<char> buf(1 << 20);
        int n;
        while ((n = gzread(g, buf.data(), (unsigned)buf.size())) > 0) data.append(buf.data(), (size_t)n);
        gzclose(g);
        if (n < 0) fail("unable to load " + path);
        return data;
    }
    fseek(f, 0, SEEK_END); long size = ftell(f); fseek(f, 0, SEEK_SET);
    data.resize((size_t)size);
    if (size > 0 && fread(&data[0], 1, (size_t)size, f) != (size_t)size) { fclose(f); fail("unable to load " + path); }
    fclose(f);
    return data;
}

static bool is_ws(char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r' || c == '\v' || c == '\f'; }

std::string read_fasta_bytes(const std::string& path) { return slurp(path); }

std::vector<FastaRecord> parse_fasta(const std::string& data, const std::string& path) {   // misc.rs:248-321
    std::vector<FastaRecord> recs;
    FastaRecord cur; bool open = false;
    auto close_record = [&]() {
        for (char& c : cur.seq) if (c >= 'a' && c <= 'z') c = (char)(c - 32);
        recs.push_back(std::move(cur)); cur = FastaRecord();
    };
    size_t pos = 0;
    while (pos < data.size()) {
        size_t eol = data.find('\n', pos);
        if (eol == std::string::npos) eol = data.size();
        size_t end = eol;
        if (end > pos && data[end - 1] == '\r') --end;           // BufRead::lines strips "\n" or "\r\n"
        if (end > pos) {
            if (data[pos] == '>') {
                if (open) close_record();
                cur.header.assign(data, pos + 1, end - pos - 1);
                size_t a = 0; while (a < cur.header.size() && is_ws(cur.header[a])) ++a;
                size_t b = a; while (b < cur.header.size() && !is_ws(cur.header[b])) ++b;
                if (a == b) fail(path + " is not correctly formatted");
                cur.name.assign(cur.header, a, b - a);
                open = true;
            } else {
                if (!open) fail(path + " is not correctly formatted");
                cur.seq.append(data, pos, end - pos);
            }
        }
        pos = eol + 1;
    }
    if (open) close_record();
    return recs;
}

void check_fasta(const std::vector<FastaRecord>& recs, const std::string& path) {   // misc.rs:174-194
    if (recs.empty()) fail(path + " contains no sequences");
    std::unordered_set<std::string> seen;
    for (auto& r : recs) {
        if (r.name.empty()) fail(path + " has an unnamed sequence");
        if (r.seq.empty()) fail(path + " has an empty sequence");
    }
    for (auto& r : recs) if (!seen.insert(r.name).second) fail(path + " has a duplicate name: " + r.name);
}

std::vector<FastaRecord> load_fasta(const std::string& path) {   // misc.rs:144-159
    struct stat st;
    if (stat(path.c_str(), &st) == 0 && st.st_size == 0) fail(path + " is an empty file");
    std::vector<FastaRecord> recs = parse_fasta(slurp(path), path);
    check_fasta(recs, path);
    return recs;
}

// ------------------------------------------------------------------------------------------------
// End repair (compress.rs:202-270).  The reference runs two regexes per sequence over every strand; here
// all 2S patterns are matched in ONE pass per strand: a pattern is k/2 wildcards next to k/2 literal bases,
// so a rolling hash of k/2-byte windows against the set of literal halves finds every candidate, and the
// regex crate's leftmost, non-overlapping `find_iter` semantics are applied per (pattern, strand).
// ------------------------------------------------------------------------------------------------
static std::string revcomp(const std::string& s) {
    std::string r(s.size(), 'N');
    for (size_t i = 0; i < s.size(); ++i) {
        char c = s[s.size() - 1 - i];
        r[i] = c == 'A' ? 'T' : c == 'T' ? 'A' : c == 'C' ? 'G' : c == 'G' ? 'C' : c == '.' ? '.' : 'N';
    }
    return r;
}

namespace {
struct Pattern { std::string literal; bool literal_last; };   // start pattern: wildcards then literal; end pattern: literal then wildcards
struct MatchTally { std::unordered_map<std::string, uint32_t> count; };

std::string best_match(const MatchTally& t) {   // find_best_match, compress.rs:239-270: fewest dots, most frequent, alphabetical
    const std::string* best = nullptr; size_t best_dots = 0; uint32_t best_n = 0;
    for (auto& kv : t.count) {
        size_t dots = (size_t)std::count(kv.first.begin(), kv.first.end(), '.');
        bool better = !best || dots < best_dots || (dots == best_dots && (kv.second > best_n || (kv.second == best_n && kv.first < *best)));
        if (better) { best = &kv.first; best_dots = dots; best_n = kv.second; }
    }
    if (!best) throw std::runtime_error("end repair: a pattern must at least match its own sequence");
    return *best;
}
}  // namespace

void sequence_end_repair(std::vector<std::string>& padded, uint32_t k, uint32_t threads) {
    const size_t m = k - 1, h = k / 2;
    if (m == 0 || padded.empty()) return;
    const size_t S = padded.size();
    std::vector<std::string> strands;                       // all_seqs, compress.rs:209 (pre-repair copies)
    strands.reserve(2 * S);
    for (auto& s : padded) { strands.push_back(s); strands.push_back(revcomp(s)); }
    std::vector<Pattern> pats(2 * S);
    for (size_t i = 0; i < S; ++i) {
        pats[2 * i] = Pattern{padded[i].substr(h, h), true};                           // first k-1 bytes: h dots + h bases
        pats[2 * i + 1] = Pattern{padded[i].substr(padded[i].size() - m, h), false};   // last k-1 bytes: h bases + h dots
    }
    const uint64_t B = 0x100000001B3ull;
    uint64_t Bh = 1; for (size_t i = 1; i < h; ++i) Bh *= B;                            // B^(h-1)
    auto hash_of = [&](const char* p) { uint64_t v = 0; for (size_t i = 0; i < h; ++i) v = v * B + (unsigned char)p[i]; return v; };
    std::unordered_map<uint64_t, std::vector<uint32_t>> by_hash;
    for (uint32_t i = 0; i < pats.size(); ++i) by_hash[hash_of(pats[i].literal.data())].push_back(i);
    std::vector<uint64_t> filter(1024, 0);                  // 64 Kbit pre-filter in front of the map
    for (auto& kv : by_hash) { uint64_t b = kv.first >> 48; filter[b >> 6] |= 1ull << (b & 63); }

    const uint32_t nt = std::max<uint32_t>(1, std::min<uint32_t>(threads, (uint32_t)strands.size()));
    std::vector<std::vector<MatchTally>> per_thread(nt, std::vector<MatchTally>(pats.size()));
    std::atomic<size_t> next_strand{0};
    auto worker = [&](uint32_t tid) {
        std::vector<MatchTally>& tally = per_thread[tid];
        std::vector<size_t> next_free(pats.size());
        for (;;) {
            const size_t si = next_strand.fetch_add(1);
            if (si >= strands.size()) return;
            const std::string& hay = strands[si];
            const size_t n = hay.size();
            if (n < m) continue;
            std::fill(next_free.begin(), next_free.end(), 0);
            uint64_t v = hash_of(hay.data());
            for (size_t j = 0;; ++j) {                      // j = start of the k/2-byte window
                const uint64_t b = v >> 48;
                if (filter[b >> 6] >> (b & 63) & 1) {
                    auto it = by_hash.find(v);
                    if (it != by_hash.end())
                        for (uint32_t pi : it->second) {
                            const Pattern& p = pats[pi];
                            if (memcmp(hay.data() + j, p.literal.data(), h) != 0) continue;
                            if (p.literal_last ? j < h : j + m > n) continue;      // the wildcard half must fit
                            const size_t start = p.literal_last ? j - h : j;
                            if (start < next_free[pi]) continue;                   // overlaps the previous match of this regex
                            next_free[pi] = start + m;
                            tally[pi].count[hay.substr(start, m)] += 1;
                        }
                }
                if (j + h >= n) break;
                v = (v - (unsigned char)hay[j] * Bh) * B + (unsigned char)hay[j + h];
            }
        }
    };
    std::vector<std::thread> pool;
    for (uint32_t t = 1; t < nt; ++t) pool.emplace_back(worker, t);
    worker(0);
    for (auto& t : pool) t.join();

    for (size_t i = 0; i < S; ++i) {
        for (int side = 0; side < 2; ++side) {
            MatchTally merged;
            for (uint32_t t = 0; t < nt; ++t) for (auto& kv : per_thread[t][2 * i + side].count) merged.count[kv.first] += kv.second;
            const std::string best = best_match(merged);
            if (side == 0) padded[i].replace(0, m, best);                          // compress.rs:223
            else padded[i].replace(padded[i].size() - m, m, best);                 // compress.rs:232
        }
    }
}

// The same end repair with the match enumeration on the device: the literal halves of the 2S patterns and their reverse
// complements are searched on the forward strands by one kernel (a hit of rc(l) at forward offset q is a hit of l on the
// reverse strand at n-q-h); leftmost non-overlapping selection, ranking and splicing stay here (a few hits per pattern).
void sequence_end_repair_device(DevicePipeline& pipe, std::vector<std::string>& padded, uint32_t k) {
    const size_t m = k - 1, h = k / 2;
    if (m == 0 || padded.empty()) return;
    const size_t S = padded.size();
    std::vector<SeqInfo> infos(S);
    std::string all;
    for (size_t i = 0; i < S; ++i) {
        SeqInfo q{}; q.start = all.size(); q.len = (uint32_t)(padded[i].size() - m); q.lead = (uint16_t)h; q.trail = (uint16_t)h; q.id = (uint16_t)(i + 1);
        infos[i] = q; all += padded[i];
    }
    // needles: distinct literals (and reverse complements), each with the patterns it stands for
    struct Use { uint32_t pattern; bool rc; };
    std::unordered_map<std::string, uint32_t> needle_of;
    std::vector<std::vector<Use>> uses;
    std::vector<uint64_t> words;
    auto add = [&](const std::string& lit, uint32_t pattern, bool is_rc) {
        auto it = needle_of.find(lit);
        if (it == needle_of.end()) {
            it = needle_of.emplace(lit, (uint32_t)uses.size()).first; uses.emplace_back();
            unsigned __int128 v = 0;
            for (char c : lit) v = (v << 2) | (unsigned)(c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : 3);
            words.push_back((uint64_t)(v >> 64)); words.push_back((uint64_t)v);
        }
        uses[it->second].push_back({pattern, is_rc});
    };
    for (size_t i = 0; i < S; ++i) {
        const std::string start_lit = padded[i].substr(h, h), end_lit = padded[i].substr(padded[i].size() - m, h);
        add(start_lit, (uint32_t)(2 * i), false); add(revcomp(start_lit), (uint32_t)(2 * i), true);
        add(end_lit, (uint32_t)(2 * i + 1), false); add(revcomp(end_lit), (uint32_t)(2 * i + 1), true);
    }
    std::vector<LiteralHit> hits;
    pipe.find_literals((const uint8_t*)all.data(), all.size(), infos.data(), (uint32_t)S, (uint32_t)h, words.data(), (uint32_t)uses.size(), hits);

    // candidates per (pattern, strand): start offset of the k-1 byte window on that strand
    struct Cand { uint32_t pattern, strand; uint64_t start; };
    std::vector<Cand> cands;
    for (const LiteralHit& hit : hits) {
        size_t si = std::upper_bound(infos.begin(), infos.end(), hit.gpos, [](uint64_t g, const SeqInfo& q) { return g < q.start; }) - infos.begin() - 1;
        const uint64_t n = padded[si].size(), q = hit.gpos - infos[si].start;
        for (const Use& u : uses[hit.needle]) {
            const uint64_t j = u.rc ? n - q - h : q;                  // literal offset on the strand the pattern matched
            const bool literal_last = (u.pattern & 1) == 0;            // start pattern: wildcards then literal
            if (literal_last ? j < h : j + m > n) continue;            // the wildcard half must fit
            cands.push_back({u.pattern, (uint32_t)(2 * si + (u.rc ? 1 : 0)), literal_last ? j - h : j});
        }
    }
    std::sort(cands.begin(), cands.end(), [](const Cand& a, const Cand& b) {
        if (a.pattern != b.pattern) return a.pattern < b.pattern;
        if (a.strand != b.strand) return a.strand < b.strand;
        return a.start < b.start; });
    std::vector<MatchTally> tally(2 * S);
    for (size_t x = 0; x < cands.size();) {
        size_t y = x; uint64_t next_free = 0;
        while (y < cands.size() && cands[y].pattern == cands[x].pattern && cands[y].strand == cands[x].strand) {
            const Cand& c = cands[y++];
            if (c.start < next_free) continue;                         // overlaps the previous match of this regex on this strand
            next_free = c.start + m;
            const std::string& fwd = padded[c.strand >> 1];
            tally[c.pattern].count[(c.strand & 1) ? revcomp(fwd.substr(fwd.size() - c.start - m, m)) : fwd.substr(c.start, m)] += 1;
        }
        x = y;
    }
    std::vector<std::string> repaired = padded;                       // matches refer to the pre-repair strands (compress.rs:209)
    for (size_t i = 0; i < S; ++i) {
        repaired[i].replace(0, m, best_match(tally[2 * i]));                                   // compress.rs:223
        repaired[i].replace(repaired[i].size() - m, m, best_match(tally[2 * i + 1]));        // compress.rs:232
    }
    padded.swap(repaired);
}

// ------------------------------------------------------------------------------------------------
LoadedInput load_sequences(const std::string& dir, uint32_t k, uint32_t max_contigs, uint32_t threads, bool verbose, DevicePipeline* device) {
    LoadedInput in;
    const std::vector<std::string> assemblies = find_all_assemblies(dir);
    in.assembly_count = assemblies.size();
    const uint32_t h = k / 2;
    size_t seq_id = 0;
    // the files are independent until ids are handed out: read and parse them on `threads` threads, then number in file order
    std::vector<std::vector<FastaRecord>> loaded(assemblies.size());
    std::vector<std::string> errors(assemblies.size());
    {
        std::atomic<size_t> next_file{0};
        auto work = [&]() {
            for (size_t f; (f = next_file.fetch_add(1)) < assemblies.size();) {
                try { loaded[f] = load_fasta(assemblies[f]); } catch (const InputError& e) { errors[f] = e.msg.empty() ? "unable to load " + assemblies[f] : e.msg; }
            }
        };
        std::vector<std::thread> pool;
        for (size_t t = 1; t < std::min<size_t>(std::max<uint32_t>(threads, 1), assemblies.size()); ++t) pool.emplace_back(work);
        work();
        for (auto& th : pool) th.join();
    }
    for (size_t file = 0; file < assemblies.size(); ++file) {
        const std::string& path = assemblies[file];
        if (!errors[file].empty()) fail(errors[file]);           // raised where the serial loop of the reference would have met it
        AssemblyDetails det; det.filename = path;
        const std::string filename = path.substr(path.rfind('/') + 1);
        for (FastaRecord& rec : loaded[file]) {
            if (rec.seq.size() < k) continue;                                      // compress.rs:109
            if (++seq_id > 32767) fail("no more than 32767 input sequences are allowed");
            std::string header;                                                    // split_whitespace().join(" "), compress.rs:115
            for (size_t a = 0; a < rec.header.size();) {
                while (a < rec.header.size() && is_ws(rec.header[a])) ++a;
                size_t b = a; while (b < rec.header.size() && !is_ws(rec.header[b])) ++b;
                if (b > a) { if (!header.empty()) header += ' '; header.append(rec.header, a, b - a); }
                a = b;
            }
            for (char c : rec.seq) if (c != 'A' && c != 'C' && c != 'G' && c != 'T') fail(filename + " contains non-ACGT characters");   // sequence.rs:40-42
            if (verbose) fprintf(stderr, " %3zu: %s %s (%zu bp)\n", seq_id, filename.c_str(), header.substr(0, header.find(' ')).c_str(), rec.seq.size());
            size_t sp = header.find(' ');
            det.contigs.push_back({header.substr(0, sp), sp == std::string::npos ? std::string() : header.substr(sp + 1), (uint64_t)rec.seq.size()});
            std::string lower = header; for (char& c : lower) if (c >= 'A' && c <= 'Z') c = (char)(c + 32);
            if (lower.find("autocycler_ignore") != std::string::npos) continue;    // sequence.rs:93-95, compress.rs:120-122
            HostSeq s; s.id = (uint16_t)seq_id; s.filename = filename; s.contig_header = header; s.length = rec.seq.size(); s.start = 0;
            in.seqs.push_back(std::move(s));
            in.padded.push_back(std::string(h, '.') + rec.seq + std::string(h, '.'));   // sequence.rs:44-46
        }
        in.details.push_back(std::move(det));
    }
    if (verbose) fprintf(stderr, "\n");
    if (in.seqs.empty()) fail("no sequences found in input assemblies");           // compress.rs:84-95
    const double mean = (double)in.seqs.size() / (double)assemblies.size();
    if (mean > (double)max_contigs) {
        char buf[256];
        snprintf(buf, sizeof buf, "the mean number of contigs per input assembly (%.1f) exceeds the allowed threshold (%u). "
                                  "Are your input assemblies fragmented or contaminated?", mean, max_contigs);
        fail(buf);
    }
    if (device) sequence_end_repair_device(*device, in.padded, k); else sequence_end_repair(in.padded, k, threads);
    return in;
}

// ------------------------------------------------------------------------------------------------
// serde_yaml 0.9 rendering of InputAssemblyMetrics (metrics.rs:65-107, 250-254)
// ------------------------------------------------------------------------------------------------
static bool yaml_needs_quotes(const std::string& s) {
    if (s.empty()) return true;
    static const char* special[] = {"~", "null", "Null", "NULL", "true", "True", "TRUE", "false", "False", "FALSE", "y", "Y", "yes", "Yes", "YES",
                                    "n", "N", "no", "No", "NO", "on", "On", "ON", "off", "Off", "OFF", ".nan", ".NaN", ".NAN", ".inf", ".Inf", ".INF",
                                    "-.inf", "-.Inf", "-.INF", "+.inf", "+.Inf", "+.INF"};
    for (const char* w : special) if (s == w) return true;
    char* end = nullptr; (void)strtod(s.c_str(), &end);
    if (end && *end == 0) return true;
    if (s.front() == ' ' || s.back() == ' ') return true;
    if (strchr("-?:,[]{}#&*!|>'\"%@`", s.front()) && !((s.front() == '-' || s.front() == '?' || s.front() == ':') && s.size() > 1 && s[1] != ' ')) return true;
    for (size_t i = 0; i < s.size(); ++i) {
        unsigned char c = (unsigned char)s[i];
        if (c < 0x20 || c == 0x7f) return true;
        if (c == ':' && (i + 1 == s.size() || s[i + 1] == ' ')) return true;
        if (c == '#' && i > 0 && s[i - 1] == ' ') return true;
    }
    return false;
}
static std::string yaml_scalar(const std::string& s) {
    if (!yaml_needs_quotes(s)) return s;
    std::string q = "'"; for (char c : s) { q += c; if (c == '\'') q += '\''; } return q + "'";
}

std::string metrics_yaml(const LoadedInput& in, uint64_t unitig_count, uint64_t unitig_total_length) {
    uint64_t total = 0; for (auto& s : in.seqs) total += s.length;
    std::string y;
    y += "input_assemblies_count: " + std::to_string(in.assembly_count) + "\n";
    y += "input_assemblies_total_contigs: " + std::to_string(in.seqs.size()) + "\n";
    y += "input_assemblies_total_length: " + std::to_string(total) + "\n";
    y += "compressed_unitig_count: " + std::to_string(unitig_count) + "\n";
    y += "compressed_unitig_total_length: " + std::to_string(unitig_total_length) + "\n";
    if (in.details.empty()) return y + "input_assembly_details: []\n";
    y += "input_assembly_details:\n";
    for (auto& a : in.details) {
        y += "- filename: " + yaml_scalar(a.filename) + "\n";
        if (a.contigs.empty()) { y += "  contigs: []\n"; continue; }
        y += "  contigs:\n";
        for (auto& c : a.contigs) {
            y += "  - name: " + yaml_scalar(c.name) + "\n";
            y += "    description: " + yaml_scalar(c.description) + "\n";
            y += "    length: " + std::to_string(c.length) + "\n";
        }
    }
    return y;
}
