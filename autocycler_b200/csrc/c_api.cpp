// extern "C" boundary of libautocycler_gpu.so (include/autocycler_gpu.h).  No exception leaves this file.
#include "../../include/autocycler_gpu.h"

#include <sched.h>
#include <dirent.h>
#include <sys/stat.h>
#include <unistd.h>
#include <cmath>
#include <zlib.h>

#include <algorithm>
#include <cerrno>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <memory>
#include <set>
#include <string>
#include <string_view>
#include <vector>

#include "backend.h"
#include "host_graph.h"
#include "host_io.h"
#include "host_cluster.h"
#include "host_trim.h"
#include "host_resolve.h"
#include "host_clean.h"
#include "host_dotplot.h"
#include "host_subsample.h"
#include "host_genome_size.h"
#include "host_depth.h"
#include "host_qv.h"
#include "host_unassembled.h"
#include "host_polish.h"
#include "host_variants.h"
#include <mutex>
#include <immintrin.h>
#include <functional>
#include <thread>
#include "commands.h"

namespace {
thread_local std::string g_error;

struct NoDevice { std::string msg; };

double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

struct PinnedBytes {     // host staging buffer for the concatenated padded strands (pinned, so the H2D copy is a DMA)
    uint8_t* p = nullptr; size_t size = 0, cap = 0;
    void append(const uint8_t* src, size_t n) {
        if (size + n > cap) {
            size_t ncap = std::max<size_t>(cap * 2, size + n + (1 << 20));
            uint8_t* q = (uint8_t*)ac_host_alloc(ncap);
            if (size) memcpy(q, p, size);
            ac_host_free(p); p = q; cap = ncap;
        }
        memcpy(p + size, src, n); size += n;
    }
    void clear() { size = 0; }
    ~PinnedBytes() { ac_host_free(p); }
};
}  // namespace

struct ac_handle {
    ac_config cfg{};
    mutable std::string err;
    std::vector<HostSeq> seqs;
    std::vector<SeqInfo> infos;
    PinnedBytes ascii;
    LoadedInput loaded;                    // only when filled by ac_load_sequences (keeps the YAML details)
    std::unique_ptr<DevicePipeline> pipe;                   // the pipeline that finishes the graph (devices[0])
    std::vector<std::unique_ptr<DevicePipeline>> peers;     // ac_config.n_devices > 1: the pipelines of devices[1..]
    // trim and resolve's alignments, cluster's distances and tree: on pipe's device and stream, made on first use
    std::unique_ptr<DeviceAlign> aligner;
    std::unique_ptr<DeviceCluster> clusterer;
    DeviceAlign& align_device() { if (!aligner) aligner.reset(new DeviceAlign(pipe->context())); return *aligner; }
    DeviceCluster& cluster_device() { if (!clusterer) clusterer.reset(new DeviceCluster(pipe->context())); return *clusterer; }
    const char* path_lines = nullptr; uint64_t path_lines_len = 0;     // ac_path_lines_render: this rank's P lines (pinned, owned by the pipeline)
    std::vector<int32_t> devices;
    PipelineResult res;
    HostGraph graph;
    std::string gfa;
    const char* gfa_ptr = nullptr; uint64_t gfa_len = 0;     // the finished file: h->gfa, or the pinned buffer the device wrote the S and L lines into
    bool uploaded = false, built = false, gfa_ready = false;
    bool fused = false;                                      // built by ac_compress: simplified on the device; the host graph is adopted on first use
    bool graph_ready = false;                                // h->graph describes the current graph
    ac_timings t{};
    uint64_t links_now = 0;
    std::string trim_yaml; bool trimmed = false;           // ac_trim: 2_trimmed.yaml
    TrimStats trim_stats;
    ClusterResult cluster; ClusterStats cluster_stats; bool clustered = false;
    ResolveResult resolve; ResolveStats resolve_stats; bool resolved = false;
};

static int set_error(const ac_handle* h, int code, const std::string& msg) {
    if (h) h->err = msg;
    g_error = msg;
    return code;
}

static int ok(const ac_handle* h) {      // a call that succeeded leaves no stale message behind (ac_last_error)
    if (h) h->err.clear();
    g_error.clear();
    return AC_OK;
}

// ---- what the commands (the ac_*_dir calls) and the getters share ----
namespace {
int check_dir(const std::string& path) {        // check_if_dir_exists (misc.rs:110-119)
    struct stat st;
    if (stat(path.c_str(), &st) != 0) return set_error(nullptr, AC_EINPUT, "directory does not exist: " + path);
    if (!S_ISDIR(st.st_mode)) return set_error(nullptr, AC_EINPUT, path + " is not a directory");
    return AC_OK;
}
int check_file(const std::string& path) {       // check_if_file_exists (misc.rs:98-107)
    struct stat st;
    if (stat(path.c_str(), &st) != 0) return set_error(nullptr, AC_EINPUT, "file does not exist: " + path);
    if (!S_ISREG(st.st_mode)) return set_error(nullptr, AC_EINPUT, path + " is not a file");
    return AC_OK;
}
int read_file(const std::string& path, std::string& text) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return set_error(nullptr, AC_EIO, "cannot read " + path);
    char buf[1 << 16]; size_t n;
    text.clear();
    while ((n = fread(buf, 1, sizeof buf, f)) > 0) text.append(buf, n);
    const bool good = !ferror(f);
    fclose(f);
    return good ? AC_OK : set_error(nullptr, AC_EIO, "cannot read " + path);
}
bool write_file(const std::string& path, std::string_view text) {      // false when the file cannot be opened, written or closed
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) return false;
    const bool good = fwrite(text.data(), 1, text.size(), f) == text.size();
    return fclose(f) == 0 && good;
}
bool make_dirs(const std::string& path) {       // create_dir_all
    struct stat st;
    if (path.empty() || stat(path.c_str(), &st) == 0) return path.empty() || S_ISDIR(st.st_mode);
    const size_t slash = path.find_last_of('/', path.size() > 1 ? path.size() - 2 : 0);
    if (slash != std::string::npos && slash > 0 && !make_dirs(path.substr(0, slash))) return false;
    return mkdir(path.c_str(), 0777) == 0 || (stat(path.c_str(), &st) == 0 && S_ISDIR(st.st_mode));
}
int remove_tree(const std::string& path) {       // everything under a directory, and the directory
    struct stat st;
    if (lstat(path.c_str(), &st) != 0) return 0;
    if (S_ISDIR(st.st_mode)) {
        DIR* d = opendir(path.c_str());
        if (!d) return -1;
        std::vector<std::string> names;
        while (dirent* e = readdir(d)) { const std::string n = e->d_name; if (n != "." && n != "..") names.push_back(n); }
        closedir(d);
        for (auto& n : names) if (remove_tree(path + "/" + n) != 0) return -1;
        return rmdir(path.c_str());
    }
    return unlink(path.c_str());
}

struct HandleDeleter { void operator()(ac_handle* h) const { ac_destroy(h); } };
using Handle = std::unique_ptr<ac_handle, HandleDeleter>;
int make_handle(int32_t device, Handle& h) {     // the handle a command makes for one device; a loaded GFA replaces its k
    ac_config cfg{}; cfg.k = 51; cfg.device = device;
    ac_handle* p = nullptr;
    const int rc = ac_create(&p, &cfg);
    h.reset(p);
    return rc;
}
int load_input_gfa(ac_handle* h, const std::string& text) {      // a malformed input GFA is one of the reference's input errors
    const int rc = ac_load_gfa(h, text.data(), text.size());
    return rc == AC_EINVAL ? AC_EINPUT : rc;
}

// A text getter: `out` NULL asks for the length only; otherwise the text is copied when `cap` holds it
int copy_text(const ac_handle* h, const std::string& text, char* out, uint64_t cap, uint64_t* length) {
    *length = text.size();
    if (!out) return ok(h);
    if (cap < text.size()) return set_error(h, AC_ERANGE, "buffer too small");
    memcpy(out, text.data(), text.size());
    return ok(h);
}

// Path x of the caller paths of ac_trim_paths / ac_bridge_best_paths: its offsets must not decrease, and every entry needs a weight
int check_path(const ac_handle* h, const int32_t* paths, const uint64_t* path_off, uint64_t x, uint64_t n_weights) {
    if (path_off[x + 1] < path_off[x]) return set_error(h, AC_EINVAL, "path offsets must not decrease");
    for (uint64_t i = path_off[x]; i < path_off[x + 1]; ++i) {
        const int32_t u = paths[i];
        const int64_t a = u < 0 ? -(int64_t)u : u;
        if (u == 0 || (uint64_t)a >= n_weights) return set_error(h, AC_EINVAL, "path entry " + std::to_string(u) + " has no weight");
    }
    return AC_OK;
}
}  // namespace

#define AC_GUARD_BEGIN try {
#define AC_GUARD_END(h) } catch (const InputError& e) { return set_error(h, AC_EINPUT, e.msg); } \
    catch (const RangeError& e) { return set_error(h, AC_ERANGE, e.msg); } \
    catch (const NoDevice& e) { return set_error(h, AC_ENODEVICE, e.msg); } \
    catch (const std::bad_alloc&) { return set_error(h, AC_ERANGE, "out of host memory"); } \
    catch (const std::exception& e) { std::string m = e.what(); \
        int code = m.find("no CUDA device") != std::string::npos ? AC_ENODEVICE : (m.find("cuda") != std::string::npos ? AC_ECUDA : AC_EINVAL); \
        return set_error(h, code, m); } \
    catch (...) { return set_error(h, AC_EINVAL, "unknown error"); }

// ac_config.n_devices > 1: the stages of SURVEY.md 8e driven from this one process.  The assemblies are sharded by file (contiguous
// blocks in the order of ac_add_sequence = sorted file order); every device builds the table of its block, then folds the other
// devices' deduplicated entries in by reading them where they lie (peer memory over NVLink: the merge kernel is the collective),
// computes adjacency and its own occurrences; devices[0] reads all occurrences the same way and finishes the graph.
static void build_on_devices(ac_handle* h, bool fused) {
    std::vector<DevicePipeline*> pipes{h->pipe.get()};
    for (auto& p : h->peers) pipes.push_back(p.get());
    const size_t N = pipes.size();
    std::vector<uint32_t> first_of_file;                     // index of the first sequence of every file
    for (size_t i = 0; i < h->seqs.size(); ++i) if (i == 0 || h->seqs[i].filename != h->seqs[i - 1].filename) first_of_file.push_back((uint32_t)i);
    first_of_file.push_back((uint32_t)h->seqs.size());
    const size_t F = first_of_file.size() - 1;
    auto on_all = [&](const std::function<void(size_t)>& work) {
        std::vector<std::thread> th; std::vector<std::exception_ptr> err(N);
        for (size_t d = 1; d < N; ++d) th.emplace_back([&, d] { try { work(d); } catch (...) { err[d] = std::current_exception(); } });
        try { work(0); } catch (...) { err[0] = std::current_exception(); }
        for (auto& t : th) t.join();
        for (auto& e : err) if (e) std::rethrow_exception(e);
    };
    std::vector<const void*> entries(N), runs(N); std::vector<uint64_t> n_entries(N), n_runs(N);
    on_all([&](size_t d) {
        pipes[d]->build_local(first_of_file[F * d / N], first_of_file[F * (d + 1) / N], true);
        entries[d] = pipes[d]->export_entries_own(&n_entries[d]);
    });
    on_all([&](size_t d) {
        for (size_t r = 0; r < N; ++r) if (r != d && n_entries[r]) pipes[d]->merge_entries(entries[r], n_entries[r]);
        pipes[d]->runs_local();
        runs[d] = pipes[d]->export_runs_own(&n_runs[d]);
    });
    pipes[0]->import_runs_from(runs.data(), n_runs.data(), (uint32_t)N);
    pipes[0]->finish(h->res, h->cfg.keep_positions != 0, fused);
}


extern "C" {

const char* ac_last_error(const ac_handle* h) { return h ? h->err.c_str() : g_error.c_str(); }

const char* ac_version(void) {
#ifdef AC_EMULATE
    return "autocycler_gpu 0.1 (host emulation build: tests only)";
#else
    return "autocycler_gpu 0.1 (sm_90a)";
#endif
}

int ac_create(ac_handle** out, const ac_config* cfg) {
    ac_handle* h = nullptr;
    AC_GUARD_BEGIN
    if (!out || !cfg) return set_error(nullptr, AC_EINVAL, "null argument");
    *out = nullptr;
    if (cfg->k < 3 || (cfg->k & 1) == 0) return set_error(nullptr, AC_EINVAL, "--kmer must be odd");          // compress.rs:58
    if (cfg->k > AC_MAX_K)
        return set_error(nullptr, AC_EINVAL, "k-mer sizes above " + std::to_string(AC_MAX_K) + " are not supported by the GPU path (there is no CPU fallback)");
    h = new ac_handle;
    h->cfg = *cfg;
    if (cfg->n_devices > 1) {
        if (!cfg->devices) { delete h; return set_error(nullptr, AC_EINVAL, "ac_config.devices is null"); }
        if (cfg->n_devices > 16) { delete h; return set_error(nullptr, AC_EINVAL, "at most 16 devices"); }
        h->devices.assign(cfg->devices, cfg->devices + cfg->n_devices);
        for (size_t a = 0; a < h->devices.size(); ++a) for (size_t b = 0; b < a; ++b) if (h->devices[a] == h->devices[b]) { delete h; return set_error(nullptr, AC_EINVAL, "ac_config.devices names a device twice"); }
        h->cfg.device = h->devices[0]; h->cfg.stream = nullptr; h->cfg.devices = nullptr;
        h->pipe.reset(new DevicePipeline(h->devices[0], nullptr));
        for (size_t d = 1; d < h->devices.size(); ++d) h->peers.emplace_back(new DevicePipeline(h->devices[d], nullptr));
        DevicePipeline::enable_peer_access(h->devices.data(), (int)h->devices.size());
    } else {
        h->cfg.n_devices = 1; h->cfg.devices = nullptr;
        h->pipe.reset(new DevicePipeline(cfg->device, cfg->stream));
    }
    *out = h;
    return ok(h);
    AC_GUARD_END(((delete h), (ac_handle*)nullptr))
}

void ac_destroy(ac_handle* h) { delete h; }

int ac_clear_sequences(ac_handle* h) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    h->seqs.clear(); h->infos.clear(); h->ascii.clear(); h->loaded = LoadedInput();
    h->uploaded = h->built = h->gfa_ready = h->fused = h->graph_ready = false;
    return ok(h);
}

int ac_add_sequence(ac_handle* h, uint16_t seq_id, const uint8_t* fwd, uint64_t n, const char* filename, const char* header) {
    if (!h || !fwd) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    const uint32_t k = h->cfg.k, half = k / 2;
    if (n < 2ull * k - 1) return set_error(h, AC_EINVAL, "padded sequence shorter than 2k-1 (contigs shorter than k are skipped by the caller, compress.rs:109)");
    if (seq_id == 0 || seq_id > 32767) return set_error(h, AC_EINVAL, "sequence id must be in 1..32767 (position.rs:21)");
    uint64_t lead = 0, trail = 0;
    while (lead < n && fwd[lead] == '.') ++lead;
    while (trail < n && fwd[n - 1 - trail] == '.') ++trail;
    if (lead > half || trail > half) return set_error(h, AC_EINVAL, "more than k/2 padding dots at a sequence end");
    for (uint64_t i = lead; i < n - trail; ++i) {
        const uint8_t c = fwd[i];
        if (c != 'A' && c != 'C' && c != 'G' && c != 'T') return set_error(h, AC_EINVAL, "sequence bytes must be ACGT with dots only at the ends");
    }
    if (n - (k - 1) > 0xFFFFFFFFull) return set_error(h, AC_ERANGE, "contig longer than Position.pos allows (position.rs:20)");
    HostSeq s; s.id = seq_id; s.filename = filename ? filename : ""; s.contig_header = header ? header : "";
    s.length = n - (k - 1); s.start = h->ascii.size;
    SeqInfo info{}; info.start = s.start; info.len = (uint32_t)s.length; info.lead = (uint16_t)lead; info.trail = (uint16_t)trail; info.id = seq_id;
    h->ascii.append(fwd, n);
    h->seqs.push_back(std::move(s)); h->infos.push_back(info);
    h->uploaded = h->built = h->gfa_ready = false;
    return ok(h);
    AC_GUARD_END(h)
}

static int upload_block(ac_handle* h, uint32_t seq_lo, uint32_t seq_hi) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    AC_GUARD_BEGIN
    if (h->seqs.empty()) return set_error(h, AC_EINPUT, "no sequences found in input assemblies");
    if (h->infos.size() != h->seqs.size()) return set_error(h, AC_EINVAL, "this handle holds a loaded graph: add sequences (after ac_clear_sequences) before ac_upload");
    {   // what save_gfa prints around every path's unitig list (unitig_graph.rs:352-360), for the device writer of the P lines
        std::string blob; std::vector<uint32_t> pre, suf;
        for (const HostSeq& q : h->seqs) {
            const std::string a = "P\t" + std::to_string(q.id) + "\t";
            std::string b = "\t*\tLN:i:" + std::to_string(q.length) + "\tFN:Z:" + q.filename + "\tHD:Z:" + q.contig_header;
            if (q.cluster > 0) b += "\tCL:i:" + std::to_string(q.cluster);
            b += "\n";
            blob += a; blob += b; pre.push_back((uint32_t)a.size()); suf.push_back((uint32_t)b.size());
        }
        h->pipe->set_path_line_texts(blob.data(), pre.data(), suf.data(), (uint32_t)h->seqs.size());
    }
    if (!h->peers.empty() && !(seq_lo == 0 && seq_hi >= h->infos.size())) return set_error(h, AC_EINVAL, "ac_upload_shard is for one device per process");
    h->pipe->upload(h->ascii.p, h->ascii.size, h->infos.data(), (uint32_t)h->infos.size(), h->cfg.k, seq_lo, seq_hi);
    for (auto& peer : h->peers) peer->upload(h->ascii.p, h->ascii.size, h->infos.data(), (uint32_t)h->infos.size(), h->cfg.k);      // every device holds every sequence (end k-mers of foreign occurrences are read from them)
    h->uploaded = true; h->built = h->gfa_ready = h->fused = h->graph_ready = false;
    return ok(h);
    AC_GUARD_END(h)
}
int ac_upload(ac_handle* h) { return upload_block(h, 0, 0xFFFFFFFFu); }
int ac_upload_shard(ac_handle* h, uint32_t seq_lo, uint32_t seq_hi) { return upload_block(h, seq_lo, seq_hi); }
int ac_strand_block(ac_handle* h, uint32_t seq_lo, uint32_t seq_hi, void** dev_ptr, uint64_t* n_bytes) {
    if (!h || !dev_ptr || !n_bytes) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    if (!h->uploaded) return set_error(h, AC_EINVAL, "ac_upload_shard must precede ac_strand_block");
    *dev_ptr = h->pipe->strand_block(seq_lo, seq_hi, n_bytes);
    return ok(h);
    AC_GUARD_END(h)
}

// The host stages edit the pinned result buffers in place, so after a graph has been processed their lines sit (dirty) in the
// CPU caches, and the next build's device->host copies onto the same lines can run at a fraction of the link rate
// (profiles/pcie_probe2.py measures it on a box).  When a handle
// is reused, the previous result is therefore flushed from the caches while the GPU is busy building the next one.
namespace {
bool cpu_has_clflushopt() { unsigned a, b, c2, d; __asm__("cpuid" : "=a"(a), "=b"(b), "=c"(c2), "=d"(d) : "a"(7), "c"(0)); return (b >> 23) & 1; }
__attribute__((target("clflushopt"))) void flush_lines_opt(const char* p, size_t n) { for (size_t i = 0; i < n; i += 64) _mm_clflushopt((void*)(p + i)); _mm_sfence(); }
void flush_lines(const char* p, size_t n) {
    static const bool opt = cpu_has_clflushopt();
    if (opt) { flush_lines_opt(p, n); return; }
    for (size_t i = 0; i < n; i += 64) _mm_clflush(p + i);
    _mm_sfence();
}
struct ResultFlusher {
    std::vector<std::thread> threads;
    void start(const PipelineResult& r) {
        if (!r.rec) return;
        const size_t U = r.n_unitigs, strands = 2 * U + 1;
        std::vector<std::pair<const char*, size_t>> ranges = {
            {(const char*)r.rec, U * sizeof(UnitigRec)}, {(const char*)r.depth, U * 4}, {(const char*)r.order, U * 4}, {r.arena, (size_t)r.arena_cap},
            {(const char*)r.next_off, strands * 4}, {(const char*)r.prev_off, strands * 4}, {(const char*)r.next, (size_t)r.n_links * 4}, {(const char*)r.prev, (size_t)r.n_links * 4},
            {(const char*)r.path, (size_t)r.n_runs * 4}, {(const char*)r.path_off, ((size_t)r.n_seqs + 1) * 8}, {(const char*)r.cands, (size_t)r.n_cands * sizeof(ExpandCandidate)},
            {(const char*)r.deps, U * sizeof(ExpandDeps)}, {(const char*)r.spec_len, (size_t)r.n_cands * 4}, {(const char*)r.fixed_start, 2 * U}};
        size_t total = 0; for (auto& x : ranges) if (x.first) total += x.second;
        const size_t T = std::max<size_t>(1, std::min<size_t>(8, total >> 20));
        for (size_t t = 0; t < T; ++t)
            threads.emplace_back([ranges, t, T] {
                for (auto& x : ranges) {
                    if (!x.first || !x.second) continue;
                    const size_t lines = (x.second + 63) / 64, a = lines * t / T, b = lines * (t + 1) / T;
                    if (b > a) flush_lines(x.first + a * 64, (b - a) * 64);
                }
            });
    }
    void join() { for (auto& th : threads) th.join(); threads.clear(); }
    ~ResultFlusher() { join(); }
};
struct CallbackScope {      // DevicePipeline::before_results holds a reference to a stack object: never let it outlive the call
    DevicePipeline* pipe;
    CallbackScope(DevicePipeline* p, std::function<void()> f) : pipe(p) { pipe->before_results = std::move(f); }
    ~CallbackScope() { pipe->before_results = nullptr; }
};
}  // namespace

static void record_timings(ac_handle* h) {
    const PipelineTimings& pt = h->res.t;
    ac_timings& t = h->t;
    t.h2d = pt.h2d; t.pack = pt.pack; t.insert = pt.insert; t.adjacency = pt.adjacency; t.boundaries = pt.boundaries; t.runs = pt.runs;
    t.unitigs = pt.unitigs; t.links = pt.links; t.seed_sort = pt.seed_sort; t.emit = pt.emit; t.d2h = pt.d2h; t.device_total = pt.total;
    t.sample = pt.sample; t.device_simplify = pt.simplify; t.device_gfa = pt.gfa;
    t.insert_kernel = pt.insert_kernel; t.trim_kernel = 0;
    uint64_t windows = 0; for (auto& s : h->seqs) windows += s.length;
    t.insert_occurrences = windows; t.table_capacity = h->res.capacity; t.table_used = h->res.n_slots_used;
    t.kernel_launches = h->pipe->kernel_launches();
    t.h2d_bytes = h->res.h2d_bytes; t.d2h_bytes = h->res.d2h_bytes;
}

static void adopt_result(ac_handle* h) {   // host graph over the device result + bookkeeping shared by ac_build / ac_build_finish / the first use after ac_compress
    const double t0 = now_ms();
    h->graph.build(h->res, h->seqs, h->cfg.k, h->cfg.keep_positions != 0);
    const double ta = now_ms();
    h->graph.check_links();
    const double tb = now_ms();
    // a plain build: the expand_repeats work list, made on the device, or (needing links and paths only) here while the sequences are
    // still being copied.  A fused build has run expand_repeats to its end: a later ac_simplify lists the candidates afresh.
    if (!h->fused && !h->graph.adopt_candidates(h->res)) h->graph.prepare_simplify();
    const double tc = now_ms();
    h->pipe->complete(h->res);
    const double t1 = now_ms();
    if (getenv("AC_HOST_PROFILE")) fprintf(stderr, "[host] adopt: graph %.2f, check_links %.2f, work list %.2f, wait for sequences %.2f ms\n", ta - t0, tb - ta, tc - tb, t1 - tc);
    if (!h->fused) { record_timings(h); h->t.host_graph = (float)(t1 - t0); h->t.host_simplify = 0; h->t.host_gfa = 0; }
    h->graph_ready = true;
}

// After ac_compress the graph arrays are still in HBM: bring them over and adopt them the first time a call needs the host graph.
static void ensure_graph(const ac_handle* ch) {
    ac_handle* h = const_cast<ac_handle*>(ch);
    if (!h->built || h->graph_ready) return;
    if (!h->fused) throw std::runtime_error("no graph on this handle");
    h->pipe->fetch_graph(h->res, h->cfg.keep_positions != 0);
    adopt_result(h);                         // simplified and renumbered on the device: the graph is taken as it is
}

// What ac_build, ac_build_finish, ac_compress and ac_compress_finish share around their device work.  A plain build adopts the result
// on the host; a fused one (simplified and written as GFA text on the device) takes only the text and the counts.
static void build_graph(ac_handle* h, bool fused, const std::function<void()>& device_work) {
    ResultFlusher flusher;
    // a fused build's graph arrays are only ever written by the host once they were fetched
    if (h->built && (!fused || h->graph_ready)) flusher.start(h->res);
    {
        CallbackScope scope(h->pipe.get(), [&flusher] { flusher.join(); });      // cleared again on every way out, exceptions included
        device_work();
    }
    if (fused) {
        h->pipe->complete(h->res);
        h->fused = true; h->graph_ready = false; h->built = true;
        h->gfa_ptr = h->res.gfa_text; h->gfa_len = h->res.gfa_bytes; h->gfa_ready = true;
        record_timings(h);
        h->t.host_graph = h->t.host_simplify = h->t.host_gfa = 0;
    } else {
        h->fused = false; h->graph_ready = false;
        adopt_result(h);
        h->built = true; h->gfa_ready = false;
    }
}

int ac_build(ac_handle* h) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    AC_GUARD_BEGIN
    if (!h->uploaded) return set_error(h, AC_EINVAL, "ac_upload must precede ac_build");
    build_graph(h, false, [h] {
        if (h->peers.empty()) h->pipe->build(h->res, h->cfg.keep_positions != 0, false);
        else build_on_devices(h, false);
    });
    return ok(h);
    AC_GUARD_END(h)
}

// compress.rs:42-47 in one call: build_kmer_graph, build_unitig_graph, simplify_unitig_graph and the text save_gfa writes, all on the
// device; only the text (and the counts compress prints) come back.  The graph itself is fetched when a later call asks for it.
int ac_compress(ac_handle* h) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    AC_GUARD_BEGIN
    if (!h->uploaded) return set_error(h, AC_EINVAL, "ac_upload must precede ac_compress");
    build_graph(h, true, [h] {
        if (h->peers.empty()) h->pipe->build(h->res, h->cfg.keep_positions != 0, true);
        else build_on_devices(h, true);
    });
    return ok(h);
    AC_GUARD_END(h)
}

// ---- multi-GPU stages: one process per GPU, the caller runs the collectives between them on device buffers ----
int ac_build_local(ac_handle* h, uint32_t seq_lo, uint32_t seq_hi, uint32_t multi) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    AC_GUARD_BEGIN
    if (!h->uploaded) return set_error(h, AC_EINVAL, "ac_upload must precede ac_build_local");
    h->built = false;
    h->pipe->build_local(seq_lo, seq_hi, multi != 0);
    return ok(h);
    AC_GUARD_END(h)
}
int ac_entries_count(ac_handle* h, uint64_t* n) {
    if (!h || !n) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    *n = h->pipe->count_entries();
    return ok(h);
    AC_GUARD_END(h)
}
int ac_entries_export(ac_handle* h, void* dst, uint64_t cap_records) {
    if (!h || !dst) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    h->pipe->export_entries(dst, cap_records);
    return ok(h);
    AC_GUARD_END(h)
}
int ac_entries_merge(ac_handle* h, const void* src, uint64_t n) {
    if (!h || (!src && n)) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    h->pipe->merge_entries(src, n);
    return ok(h);
    AC_GUARD_END(h)
}
int ac_runs_local(ac_handle* h, uint64_t* n_runs) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    AC_GUARD_BEGIN
    h->pipe->runs_local();
    if (n_runs) *n_runs = h->pipe->local_runs();
    return ok(h);
    AC_GUARD_END(h)
}
int ac_runs_export(ac_handle* h, void* dst, uint64_t cap_records) {
    if (!h || !dst) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    h->pipe->export_runs(dst, cap_records);
    return ok(h);
    AC_GUARD_END(h)
}
int ac_runs_import(ac_handle* h, const void* src, uint64_t n) {
    if (!h || !src) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    h->pipe->import_runs(src, n);
    return ok(h);
    AC_GUARD_END(h)
}
int ac_runs_import_padded(ac_handle* h, const void* src, uint64_t stride_records, const uint64_t* counts, uint32_t n_ranks) {
    if (!h || !src || !counts) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    h->pipe->import_runs_padded(src, stride_records, counts, n_ranks);
    return ok(h);
    AC_GUARD_END(h)
}
// ac_compress on the rank that imported every rank's occurrences: simplify_structure and the GFA text on the device as well
static int compress_finish(ac_handle* h, bool split_paths) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    AC_GUARD_BEGIN
    build_graph(h, true, [h, split_paths] { h->pipe->finish(h->res, h->cfg.keep_positions != 0, true, split_paths); });
    return ok(h);
    AC_GUARD_END(h)
}
int ac_compress_finish(ac_handle* h) { return compress_finish(h, false); }
int ac_compress_finish_split(ac_handle* h) { return compress_finish(h, true); }
int ac_path_tokens_export(ac_handle* h, void* dst, uint64_t stride_tokens, const uint64_t* counts, uint32_t n_ranks) {
    if (!h || !dst || !counts) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    h->pipe->export_path_tokens(dst, stride_tokens, counts, n_ranks);
    return ok(h);
    AC_GUARD_END(h)
}
int ac_path_lines_render(ac_handle* h, const void* tokens, uint64_t n_tokens) {
    if (!h || (!tokens && n_tokens)) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    h->path_lines = nullptr; h->path_lines_len = 0;
    h->pipe->render_path_lines(tokens, n_tokens, &h->path_lines, &h->path_lines_len);
    return ok(h);
    AC_GUARD_END(h)
}
int ac_path_lines_data(ac_handle* h, const char** data, uint64_t* n_bytes) {
    if (!h || !data || !n_bytes) return set_error(h, AC_EINVAL, "null argument");
    *data = h->path_lines; *n_bytes = h->path_lines_len;
    return ok(h);
}
int ac_build_finish(ac_handle* h) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    AC_GUARD_BEGIN
    build_graph(h, false, [h] { h->pipe->finish(h->res, h->cfg.keep_positions != 0); });
    return ok(h);
    AC_GUARD_END(h)
}

int ac_simplify(ac_handle* h) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    AC_GUARD_BEGIN
    if (!h->built) return set_error(h, AC_EINVAL, "ac_build must precede ac_simplify");
    if (h->fused && !h->graph_ready) return ok(h);        // ac_compress has simplified the graph already
    const double t0 = now_ms();
    h->graph.simplify_structure();
    h->t.host_simplify = (float)(now_ms() - t0);
    h->gfa_ready = false;
    return ok(h);
    AC_GUARD_END(h)
}

int ac_merge_linear_paths(ac_handle* h, int use_paths) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    AC_GUARD_BEGIN
    if (!h->built) return set_error(h, AC_EINVAL, "ac_build must precede ac_merge_linear_paths");
    ensure_graph(h);
    h->graph.merge_linear_paths(use_paths != 0);
    h->gfa_ready = false;
    return ok(h);
    AC_GUARD_END(h)
}

// One process per GPU, kept on the CPU socket that GPU hangs off (what `numactl --cpunodebind` does): pinned buffers allocated
// afterwards are local to the DMA engine and to the host threads that edit them.  Changes the calling thread's affinity mask (threads created later inherit it); opt-in for that reason.
int ac_bind_host_to_device(int32_t device) {
    AC_GUARD_BEGIN
#ifdef AC_EMULATE
    (void)device;
    return set_error(nullptr, AC_ENODEVICE, "no CUDA device in the emulation build");
#else
    char bus[64] = {0};
    if (cudaDeviceGetPCIBusId(bus, (int)sizeof bus, device) != cudaSuccess) { cudaGetLastError(); return set_error(nullptr, AC_ENODEVICE, "cannot query the PCI bus id of the device"); }
    std::string id(bus);
    for (char& ch : id) ch = (char)tolower((unsigned char)ch);
    if (id.size() > 12 && id.find(':') == 8) id = id.substr(4);                      // an 8-digit PCI domain where sysfs has 4
    FILE* f = fopen(("/sys/bus/pci/devices/" + id + "/numa_node").c_str(), "r");
    int node = -1;
    if (f) { if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f); }
    if (node < 0) return set_error(nullptr, AC_EINVAL, "the device reports no NUMA node");
    f = fopen(("/sys/devices/system/node/node" + std::to_string(node) + "/cpulist").c_str(), "r");
    if (!f) return set_error(nullptr, AC_EINVAL, "cannot read the CPU list of the device's NUMA node");
    char list[4096] = {0};
    const bool got = fgets(list, sizeof list, f) != nullptr;
    fclose(f);
    if (!got) return set_error(nullptr, AC_EINVAL, "cannot read the CPU list of the device's NUMA node");
    cpu_set_t now, want; CPU_ZERO(&want);
    if (sched_getaffinity(0, sizeof now, &now) != 0) return set_error(nullptr, AC_EINVAL, "sched_getaffinity failed");
    int count = 0;
    for (char* tok = strtok(list, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
        int a = 0, b = 0;
        const int n = sscanf(tok, "%d-%d", &a, &b);
        if (n < 1) continue;
        if (n == 1) b = a;
        for (int cpu = a; cpu <= b && cpu < CPU_SETSIZE; ++cpu) if (CPU_ISSET(cpu, &now)) { CPU_SET(cpu, &want); ++count; }
    }
    if (count < 8) return set_error(nullptr, AC_EINVAL, "fewer than 8 usable CPUs on the device's NUMA node: affinity left alone");
    if (sched_setaffinity(0, sizeof want, &want) != 0) return set_error(nullptr, AC_EINVAL, "sched_setaffinity failed");
    return node;
#endif
    AC_GUARD_END(nullptr)
}

int ac_load_gfa(ac_handle* h, const char* gfa_text, uint64_t length) {
    if (!h || !gfa_text) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    h->built = false; h->gfa_ready = false; h->uploaded = false; h->fused = false; h->graph_ready = false;
    h->seqs.clear(); h->infos.clear(); h->ascii.clear(); h->loaded = LoadedInput(); h->res = PipelineResult(); h->t = ac_timings{};   // a loaded graph has no sequence bytes: ac_upload / ac_build need ac_add_sequence again
    h->trimmed = false; h->trim_yaml.clear();
    h->clustered = false; h->cluster = ClusterResult();
    h->resolved = false; h->resolve = ResolveResult();
    h->graph.load_gfa(gfa_text, (size_t)length, h->seqs);
    h->cfg.k = h->graph.k;
    h->built = true; h->graph_ready = true;
    return ok(h);
    AC_GUARD_END(h)
}

// cluster.rs:132-151: distances[a][b] = 1 - (length of the unitigs shared by a's and b's paths) / (length of a's unitigs), in the order
// of the handle's sequences.  The shared lengths are whole numbers found on the device; the one division per pair is done here in
// f64 exactly as the reference does it.
int ac_pairwise_distances(ac_handle* h, double* out, uint64_t cap) {
    if (!h || !out) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    if (!h->built) return set_error(h, AC_EINVAL, "a graph must be built or loaded before ac_pairwise_distances");
    ensure_graph(h);
    const HostGraph& g = h->graph;
    const uint64_t S = h->seqs.size();
    if (cap < S * S) return set_error(h, AC_ERANGE, "buffer too small");
    std::vector<uint32_t> len(g.U);
    for (uint32_t u = 0; u < g.U; ++u) len[u] = g.rec[u].len;
    std::vector<uint64_t> shared(S * S);
    h->cluster_device().pair_shared_lengths(g.path, g.path_off, (uint32_t)S, len.data(), g.U, shared.data());
    for (uint64_t a = 0; a < S; ++a) {
        const double a_len = (double)(uint32_t)shared[a * S + a];                    // the reference sums u32 lengths, then converts
        for (uint64_t b = 0; b < S; ++b) out[a * S + b] = 1.0 - ((double)shared[a * S + b] / a_len);
    }
    return ok(h);
    AC_GUARD_END(h)
}

// save_distance_matrix (cluster.rs:160-176): count, then one row per sequence: its Display form (sequence.rs:112-135) and the
// distances with eight decimals.
int ac_distance_matrix_text(ac_handle* h, char* out, uint64_t cap, uint64_t* length) {
    if (!h || !length) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    const uint64_t S = h->seqs.size();
    std::vector<double> d(std::max<uint64_t>(1, S * S));
    const int rc = ac_pairwise_distances(h, d.data(), S * S);
    if (rc != AC_OK) return rc;
    return copy_text(h, distance_matrix_text(h->seqs, d.data()), out, cap, length);
    AC_GUARD_END(h)
}

int ac_renumber_unitigs(ac_handle* h) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    AC_GUARD_BEGIN
    if (!h->built) return set_error(h, AC_EINVAL, "ac_build must precede ac_renumber_unitigs");
    ensure_graph(h);
    h->graph.renumber();
    h->gfa_ready = false;
    return ok(h);
    AC_GUARD_END(h)
}

int ac_counts_get(const ac_handle* h, ac_counts* out) {
    if (!h || !out) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    if (!h->built) return set_error(h, AC_EINVAL, "ac_build must precede ac_counts_get");
    memset(out, 0, sizeof *out);
    if (h->fused && !h->graph_ready) {       // straight from the device: what compress prints (compress.rs:152, unitig_graph.rs:509-516)
        const PipelineResult& r = h->res;
        out->n_kmers = 2 * r.n_slots_used; out->n_unitigs = r.n_unitigs; out->n_links = r.links_single;
        out->total_length = r.length_after; out->seq_bytes = r.length_after; out->length_before_simplify = r.length_before;
        out->n_next = r.n_links; out->n_sequences = h->seqs.size(); out->n_path_steps = r.n_runs;
        if (h->cfg.keep_positions) { out->n_fwd_pos = r.n_runs; out->n_rev_pos = r.n_runs; }
        return ok(h);
    }
    const HostGraph& g = h->graph;
    out->length_before_simplify = h->res.length_before;
    out->n_kmers = 2 * h->res.n_slots_used;
    out->n_unitigs = g.U;
    out->n_links = g.link_count_single();
    out->total_length = g.total_length();
    out->seq_bytes = out->total_length;
    out->n_fwd_pos = g.fpos.size(); out->n_rev_pos = g.rpos.size();
    out->n_next = g.n_links;
    out->n_sequences = h->seqs.size();
    out->n_path_steps = g.n_path;
    return ok(h);
    AC_GUARD_END(h)
}

int ac_unitigs_copy(const ac_handle* h, ac_unitigs* o) {
    if (!h || !o) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    if (!h->built) return set_error(h, AC_EINVAL, "ac_build must precede ac_unitigs_copy");
    ensure_graph(h);
    const HostGraph& g = h->graph;
    const bool have_pos = !g.fpos_off.empty();
    if ((o->fpos_off || o->fpos || o->rpos_off || o->rpos) && !have_pos) return set_error(h, AC_EINVAL, "positions need ac_config.keep_positions");
    uint64_t so = 0, fo = 0, ro = 0, no = 0;
    for (uint32_t n = 0; n < g.U; ++n) {
        const uint32_t u = g.order[n];
        if (o->number) o->number[n] = g.number[u];
        if (o->depth) o->depth[n] = g.depth_of(u);
        if (o->seq_off) o->seq_off[n] = so;
        if (o->seq) memcpy(o->seq + so, g.seq_ptr(u), g.rec[u].len);
        so += g.rec[u].len;
        if (o->fpos_off) o->fpos_off[n] = fo;
        if (o->rpos_off) o->rpos_off[n] = ro;
        if (have_pos) {
            for (uint64_t x = g.fpos_off[u]; x < g.fpos_off[u + 1]; ++x) { if (o->fpos) o->fpos[fo] = (uint32_t)(g.fpos[x] >> 16); if (o->fpos_id_strand) o->fpos_id_strand[fo] = (uint16_t)(g.fpos[x] & 0xFFFF); ++fo; }
            for (uint64_t x = g.rpos_off[u]; x < g.rpos_off[u + 1]; ++x) { if (o->rpos) o->rpos[ro] = (uint32_t)(g.rpos[x] >> 16); if (o->rpos_id_strand) o->rpos_id_strand[ro] = (uint16_t)(g.rpos[x] & 0xFFFF); ++ro; }
        }
        for (uint32_t rev = 0; rev < 2; ++rev) {
            if (o->next_off) o->next_off[2 * (size_t)n + rev] = no;
            const UStrand from = us_make(u, rev != 0);
            for (uint32_t x = g.next_off[from]; x < g.next_off[from + 1]; ++x) {
                if (o->next) { const int32_t num = (int32_t)g.number[us_index(g.next[x])]; o->next[no] = us_reverse(g.next[x]) ? -num : num; }
                ++no;
            }
        }
    }
    if (o->seq_off) o->seq_off[g.U] = so;
    if (o->fpos_off) o->fpos_off[g.U] = fo;
    if (o->rpos_off) o->rpos_off[g.U] = ro;
    if (o->next_off) o->next_off[2 * (size_t)g.U] = no;
    return ok(h);
    AC_GUARD_END(h)
}

int ac_path_copy(const ac_handle* h, uint64_t seq_index, int32_t* out, uint64_t cap, uint64_t* n) {
    if (!h || !n) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    if (h->built) ensure_graph(h);
    const HostGraph& g = h->graph;
    if (!h->built || seq_index >= g.n_seqs) return set_error(h, AC_EINVAL, "no such sequence");
    const uint64_t a = g.path_off[seq_index], b = g.path_off[seq_index + 1];
    *n = b - a;
    if (!out) return ok(h);
    if (cap < b - a) return set_error(h, AC_ERANGE, "path buffer too small");
    for (uint64_t x = a; x < b; ++x) { const int32_t num = (int32_t)g.number[us_index(g.path[x])]; out[x - a] = us_reverse(g.path[x]) ? -num : num; }
    return ok(h);
    AC_GUARD_END(h)
}

int ac_gfa_size(ac_handle* h, uint64_t* n_bytes) {
    if (!h || !n_bytes) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    if (!h->built) return set_error(h, AC_EINVAL, "ac_build must precede ac_gfa_size");
    if (!h->gfa_ready) {
        const double t0 = now_ms();
        ensure_graph(h);
        h->graph.gfa_text(h->seqs, h->gfa);
        h->gfa_ptr = h->gfa.data(); h->gfa_len = h->gfa.size();
        h->t.host_gfa = (float)(now_ms() - t0);
        h->gfa_ready = true;
        if (getenv("AC_HOST_PROFILE")) {
            const HostProfile& p = h->graph.prof;
            fprintf(stderr, "[host] adopt %.1f renumber(total) %.1f expand %.1f (%d passes; candidates %.1f, +compare %.1f, pass1 %.1f) gfa %.1f ms; U=%u\n",
                    p.adopt, p.renumber, p.expand, p.passes, p.candidates, p.compare, p.pass1, (double)h->t.host_gfa, h->graph.U);
        }
    }
    *n_bytes = h->gfa_len;
    return ok(h);
    AC_GUARD_END(h)
}

int ac_gfa_data(ac_handle* h, const char** data, uint64_t* n_bytes) {   // borrowed pointer, valid until the next call on this handle
    if (!data) return set_error(h, AC_EINVAL, "null argument");
    int rc = ac_gfa_size(h, n_bytes);
    if (rc != AC_OK) return rc;
    *data = h->gfa_ptr;
    return ok(h);
}

int ac_gfa_copy(ac_handle* h, char* buf, uint64_t cap) {
    uint64_t n = 0;
    int rc = ac_gfa_size(h, &n);
    if (rc != AC_OK) return rc;
    if (!buf || cap < n) return set_error(h, AC_ERANGE, "GFA buffer too small");
    memcpy(buf, h->gfa_ptr, n);
    return ok(h);
}

int ac_timings_get(const ac_handle* h, ac_timings* out) {
    if (!h || !out) return set_error(h, AC_EINVAL, "null argument");
    *out = h->t;
    out->kernel_launches = h->pipe->kernel_launches();
    return ok(h);
}

int ac_load_sequences(ac_handle* h, const char* dir, uint32_t max_contigs, uint32_t threads, uint64_t* assembly_count) {
    if (!h || !dir) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    ac_clear_sequences(h);
    // end repair runs on the device unless its k/2-base literals are longer than the scan kernel's two key words (k > 129)
    const bool device_repair = h->cfg.k / 2 <= 64;
    LoadedInput in = load_sequences(dir, h->cfg.k, max_contigs, threads ? threads : 1, false, device_repair ? h->pipe.get() : nullptr);
    for (size_t i = 0; i < in.seqs.size(); ++i) {
        int rc = ac_add_sequence(h, in.seqs[i].id, (const uint8_t*)in.padded[i].data(), in.padded[i].size(),
                                 in.seqs[i].filename.c_str(), in.seqs[i].contig_header.c_str());
        if (rc != AC_OK) return rc;
    }
    if (assembly_count) *assembly_count = in.assembly_count;
    in.padded.clear(); in.padded.shrink_to_fit();
    h->loaded = std::move(in);
    return ok(h);
    AC_GUARD_END(h)
}

int ac_sequence_get(const ac_handle* h, uint64_t index, uint16_t* seq_id, uint64_t* length, char* fwd, uint64_t cap_fwd,
                    char* filename, uint64_t cap_fn, char* header, uint64_t cap_hd) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    if (index >= h->seqs.size()) return set_error(h, AC_EINVAL, "no such sequence");
    const HostSeq& s = h->seqs[index];
    const uint64_t padded = s.length + h->cfg.k - 1;
    if (seq_id) *seq_id = s.id;
    if (length) *length = s.length;
    if (fwd) {
        if (!h->ascii.p || h->infos.empty()) return set_error(h, AC_EINVAL, "this handle holds a loaded graph: its sequences have no bytes (use ac_sequence_reconstruct)");
        if (cap_fwd < padded + 1) return set_error(h, AC_ERANGE, "buffer too small");
        memcpy(fwd, h->ascii.p + s.start, padded); fwd[padded] = 0;
    }
    if (filename) { if (cap_fn < s.filename.size() + 1) return set_error(h, AC_ERANGE, "buffer too small"); memcpy(filename, s.filename.c_str(), s.filename.size() + 1); }
    if (header) { if (cap_hd < s.contig_header.size() + 1) return set_error(h, AC_ERANGE, "buffer too small"); memcpy(header, s.contig_header.c_str(), s.contig_header.size() + 1); }
    return ok(h);
}

// reconstruct_original_sequence / get_sequence_from_path (unitig_graph.rs:383-400): the unitig strands of the sequence's
// path, concatenated; equals the input contig (tests.rs:114-127).
int ac_sequence_reconstruct(const ac_handle* h, uint64_t index, char* out, uint64_t cap, uint64_t* length) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    AC_GUARD_BEGIN
    if (!h->built) return set_error(h, AC_EINVAL, "ac_build must precede ac_sequence_reconstruct");
    if (index >= h->seqs.size()) return set_error(h, AC_EINVAL, "no such sequence");
    ensure_graph(h);
    const HostGraph& g = h->graph;
    uint64_t total = 0;
    for (uint64_t x = g.path_off[index]; x < g.path_off[index + 1]; ++x) total += g.rec[us_index(g.path[x])].len;
    if (length) *length = total;
    if (!out) return ok(h);
    if (cap < total) return set_error(h, AC_ERANGE, "buffer too small");
    char* p = out;
    for (uint64_t x = g.path_off[index]; x < g.path_off[index + 1]; ++x) {
        const UStrand s = g.path[x]; const uint32_t n = g.rec[us_index(s)].len; const char* src = g.seq_ptr(us_index(s));
        if (!us_reverse(s)) memcpy(p, src, n);
        else for (uint32_t j = 0; j < n; ++j) { const char b = src[n - 1 - j]; p[j] = b == 'A' ? 'T' : b == 'C' ? 'G' : b == 'G' ? 'C' : b == 'T' ? 'A' : b; }
        p += n;
    }
    return ok(h);
    AC_GUARD_END(h)
}

int ac_compress_dir(const char* assemblies_dir, const char* autocycler_dir, uint32_t k, uint32_t max_contigs, uint32_t threads,
                    int32_t device, int32_t verbose) {
    return ac_compress_dir_devices(assemblies_dir, autocycler_dir, k, max_contigs, threads, &device, 1, verbose);
}

int ac_compress_dir_devices(const char* assemblies_dir, const char* autocycler_dir, uint32_t k, uint32_t max_contigs, uint32_t threads,
                            const int32_t* devices, int32_t n_devices, int32_t verbose) {
    if (!assemblies_dir || !autocycler_dir || !devices || n_devices < 1) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    // check_settings, compress.rs:53-62
    int rc = check_dir(assemblies_dir);
    if (rc != AC_OK) return rc;
    struct stat st;
    if (stat(autocycler_dir, &st) == 0 && !S_ISDIR(st.st_mode)) return set_error(nullptr, AC_EINPUT, std::string(autocycler_dir) + " exists but is not a directory");
    if (k < 11) return set_error(nullptr, AC_EINPUT, "--kmer cannot be less than 11");
    if (k > 501) return set_error(nullptr, AC_EINPUT, "--kmer cannot be greater than 501");
    if (k % 2 == 0) return set_error(nullptr, AC_EINPUT, "--kmer must be odd");
    if (threads < 1) return set_error(nullptr, AC_EINPUT, "--threads cannot be less than 1");
    if (threads > 100) return set_error(nullptr, AC_EINPUT, "--threads cannot be greater than 100");
    if (k > AC_MAX_K) return set_error(nullptr, AC_EINPUT, "--kmer above " + std::to_string(AC_MAX_K) + " is not supported by this build of the GPU path (there is no CPU fallback)");
    ac_config cfg{}; cfg.k = k; cfg.device = devices[0]; cfg.stream = nullptr; cfg.keep_positions = 0; cfg.n_devices = n_devices; cfg.devices = devices;
    ac_handle* p = nullptr;
    if ((rc = ac_create(&p, &cfg)) != AC_OK) return rc;
    Handle h(p);
    make_dirs(autocycler_dir);           // a directory that cannot be made shows as "cannot write" below
    uint64_t assemblies = 0;
    const double t0 = now_ms();
    if ((rc = ac_load_sequences(h.get(), assemblies_dir, max_contigs, threads, &assemblies)) != AC_OK) return rc;
    const double t1 = now_ms();
    if (verbose) fprintf(stderr, "%zu sequence%s loaded from %llu assembl%s\n\n", h->seqs.size(), h->seqs.size() == 1 ? "" : "s",
                         (unsigned long long)assemblies, assemblies == 1 ? "y" : "ies");
    if ((rc = ac_upload(h.get())) != AC_OK || (rc = ac_compress(h.get())) != AC_OK) return rc;
    ac_counts c{};
    ac_counts_get(h.get(), &c);
    // simplify_structure moves bases between unitigs: the counts stay, the total length shrinks (print_basic_graph_info, unitig_graph.rs:509-516)
    if (verbose) fprintf(stderr, "Graph contains %llu k-mers\n\n%llu unitig%s, %llu link%s\ntotal length: %llu bp\n\n", (unsigned long long)c.n_kmers,
                         (unsigned long long)c.n_unitigs, c.n_unitigs == 1 ? "" : "s", (unsigned long long)c.n_links, c.n_links == 1 ? "" : "s",
                         (unsigned long long)c.length_before_simplify);
    if (verbose) fprintf(stderr, "%llu unitig%s, %llu link%s\ntotal length: %llu bp\n\n", (unsigned long long)c.n_unitigs, c.n_unitigs == 1 ? "" : "s",
                         (unsigned long long)c.n_links, c.n_links == 1 ? "" : "s", (unsigned long long)c.total_length);
    uint64_t n = 0;
    if ((rc = ac_gfa_size(h.get(), &n)) != AC_OK) return rc;
    const std::string out_gfa = std::string(autocycler_dir) + "/input_assemblies.gfa", out_yaml = std::string(autocycler_dir) + "/input_assemblies.yaml";
    if (!write_file(out_gfa, std::string_view(h->gfa_ptr, h->gfa_len))) return set_error(nullptr, AC_EIO, "cannot write " + out_gfa);
    if (!write_file(out_yaml, metrics_yaml(h->loaded, c.n_unitigs, c.total_length))) return set_error(nullptr, AC_EIO, "cannot write " + out_yaml);
    if (verbose) {
        const ac_timings& t = h->t;
        fprintf(stderr, "Compressed unitig graph: %s\nInput assembly stats:    %s\n", out_gfa.c_str(), out_yaml.c_str());
        fprintf(stderr, "load+repair %.1f ms | h2d %.2f pack %.2f insert %.2f adjacency %.2f boundaries %.2f runs %.2f unitigs %.2f links %.2f d2h %.2f ms"
                        " simplify %.2f gfa %.2f | host graph %.1f simplify %.1f gfa %.1f ms | total %.1f ms\n\n",
                t1 - t0, t.h2d, t.pack, t.insert, t.adjacency, t.boundaries, t.runs, t.unitigs, t.links, t.d2h, t.device_simplify, t.device_gfa, t.host_graph, t.host_simplify, t.host_gfa, now_ms() - t0);
    }
    return ok(h.get());
    AC_GUARD_END(nullptr)
}

// `autocycler decompress` (decompress.rs:27-114): reconstructs every input contig from its path and writes them back per
// original file (FASTA, gzip when the name ends in .gz) and/or into one FASTA file.
int ac_decompress_gfa(const char* in_gfa, const char* out_dir, const char* out_file, int32_t device, int32_t verbose) {
    if (!in_gfa) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    int rc = check_file(in_gfa);
    if (rc != AC_OK) return rc;
    struct stat st;
    const bool to_dir = out_dir && *out_dir, to_file = out_file && *out_file;
    if (!to_dir && !to_file) return set_error(nullptr, AC_EINPUT, "either --out_dir or --out_file is required");                  // decompress.rs:45-47
    if (to_dir && stat(out_dir, &st) == 0 && !S_ISDIR(st.st_mode)) return set_error(nullptr, AC_EINPUT, std::string(out_dir) + " exists but is not a directory");
    std::string text; Handle h;
    if ((rc = read_file(in_gfa, text)) != AC_OK || (rc = make_handle(device, h)) != AC_OK || (rc = load_input_gfa(h.get(), text)) != AC_OK) return rc;
    if (verbose) {
        ac_counts c{}; ac_counts_get(h.get(), &c);
        fprintf(stderr, "%llu unitig%s, %llu link%s\ntotal length: %llu bp\n\n", (unsigned long long)c.n_unitigs, c.n_unitigs == 1 ? "" : "s",
                (unsigned long long)c.n_links, c.n_links == 1 ? "" : "s", (unsigned long long)c.total_length);
    }
    // reconstruct_original_sequences (unitig_graph.rs:362-370): per filename, in sequence order; filenames sorted when written
    std::vector<std::string> seqs(h->seqs.size());
    for (size_t i = 0; i < h->seqs.size(); ++i) {
        uint64_t n = 0;
        if ((rc = ac_sequence_reconstruct(h.get(), i, nullptr, 0, &n)) != AC_OK) return rc;
        if (n != h->seqs[i].length) return set_error(nullptr, AC_EINPUT, "reconstructed sequence does not have expected length");   // unitig_graph.rs:386
        seqs[i].resize(n);
        if (n && (rc = ac_sequence_reconstruct(h.get(), i, &seqs[i][0], n, &n)) != AC_OK) return rc;
    }
    std::vector<std::string> names;
    for (auto& s : h->seqs) names.push_back(s.filename);
    std::sort(names.begin(), names.end()); names.erase(std::unique(names.begin(), names.end()), names.end());
    auto first_word = [](const std::string& hd) { return hd.substr(0, hd.find(' ')); };
    if (to_dir) {
        make_dirs(out_dir);              // as in compress: a failure shows as "cannot write"
        for (const std::string& name : names) {
            const std::string path = std::string(out_dir) + "/" + name;
            if (verbose) fprintf(stderr, "%s:\n", path.c_str());
            std::string body;
            for (size_t i = 0; i < h->seqs.size(); ++i)
                if (h->seqs[i].filename == name) {
                    if (verbose) fprintf(stderr, "  %s (%zu bp)\n", first_word(h->seqs[i].contig_header).c_str(), seqs[i].size());
                    body += ">" + h->seqs[i].contig_header + "\n" + seqs[i] + "\n";
                }
            const bool gz = path.size() >= 3 && path.compare(path.size() - 3, 3, ".gz") == 0;       // decompress.rs:96
            if (gz) {
                gzFile g = gzopen(path.c_str(), "wb");
                if (!g || (body.size() && gzwrite(g, body.data(), (unsigned)body.size()) != (int)body.size())) { if (g) gzclose(g); return set_error(nullptr, AC_EIO, "cannot write " + path); }
                gzclose(g);
            } else if (!write_file(path, body)) {
                return set_error(nullptr, AC_EIO, "cannot write " + path);
            }
            if (verbose) fprintf(stderr, "\n");
        }
    }
    if (to_file) {   // decompress.rs:116-137
        if (verbose) fprintf(stderr, "%s:\n", out_file);
        std::string body;
        for (const std::string& name : names) {
            std::string clean = name; for (char& ch : clean) if (ch == ' ') ch = '_';
            for (size_t i = 0; i < h->seqs.size(); ++i)
                if (h->seqs[i].filename == name) {
                    if (verbose) fprintf(stderr, "  %s__%s (%zu bp)\n", name.c_str(), first_word(h->seqs[i].contig_header).c_str(), seqs[i].size());
                    body += ">" + clean + "__" + h->seqs[i].contig_header + "\n" + seqs[i] + "\n";
                }
        }
        if (!write_file(out_file, body)) return set_error(nullptr, AC_EIO, std::string("cannot write ") + out_file);
        if (verbose) fprintf(stderr, "\n");
    }
    return ok(h.get());
    AC_GUARD_END(nullptr)
}

// ---- what ac_trim_dirs and ac_resolve_dirs share ----
namespace {
// Every directory's report, kept in memory while the clusters go through the phases together and printed to stderr in argument order
// when the call returns, whether it succeeded or not.
struct DirReports {
    struct Report { char* buf = nullptr; size_t len = 0; FILE* f = nullptr; };
    std::vector<Report> r;
    explicit DirReports(uint32_t n) : r(n) {
        for (Report& x : r) if (!(x.f = open_memstream(&x.buf, &x.len))) throw std::bad_alloc();
    }
    FILE* operator[](size_t i) const { return r[i].f; }
    ~DirReports() {
        for (Report& x : r) { fclose(x.f); fwrite(x.buf, 1, x.len, stderr); free(x.buf); }
        fflush(stderr);
    }
};

// The cluster directories of a batch: none null, and none given twice (the two runs would write the same files).  Called per directory,
// after its existence check, so the error order is the single call's.
struct DirSet {
    std::set<std::string> seen;
    int add(const std::string& dir) {
        char* r = realpath(dir.c_str(), nullptr);
        const std::string key = r ? r : dir;
        free(r);
        if (!seen.insert(key).second) return set_error(nullptr, AC_EINPUT, "cluster directory given twice: " + dir);
        return AC_OK;
    }
};

// load_input_gfa's codes and messages, into a graph of the caller's
int load_graph(const std::string& text, HostGraph& g, std::vector<HostSeq>& seqs) {
    const int rc = [&]() -> int {
        AC_GUARD_BEGIN
        g.load_gfa(text.data(), text.size(), seqs);
        return AC_OK;
        AC_GUARD_END(nullptr)
    }();
    return rc == AC_EINVAL ? AC_EINPUT : rc;
}

void fill_batch_info(const AlignBatch& b, ac_batch_info* info) {
    if (!info) return;
    info->clusters = b.clusters; info->launches = b.launches; info->jobs = b.jobs; info->cells = b.cells; info->buffer_bytes = b.buffer_bytes;
    info->kernel_ms = b.kernel_ms;
}

// trim.rs:36-67 for n directories; ac_trim_dir is n = 1
int trim_dirs(const char* const* cluster_dirs, uint32_t n, double min_identity, uint32_t max_unitigs, double mad, uint32_t threads, int32_t device,
              int32_t verbose, ac_batch_info* info) {
    if (!cluster_dirs || n == 0) return set_error(nullptr, AC_EINVAL, n == 0 ? "no cluster directory" : "null argument");
    for (uint32_t i = 0; i < n; ++i) if (!cluster_dirs[i]) return set_error(nullptr, AC_EINVAL, "null argument");
    if (info) *info = ac_batch_info{};
    AC_GUARD_BEGIN
    DirReports reports(n);
    DirSet dirs;
    std::vector<HostGraph> graphs(n);
    std::vector<std::vector<HostSeq>> seqs(n);
    Handle h;
    for (uint32_t i = 0; i < n; ++i) {
        FILE* log = reports[i];
        const std::string dir = cluster_dirs[i], in_gfa = dir + "/1_untrimmed.gfa";
        if (verbose & AC_VERBOSE_BANNER)
            fprintf(log, "\nStarting autocycler trim (%s)\n\nSettings:\n  --cluster_dir %s\n  --min_identity %g\n  --max_unitigs %u\n  --mad %g\n  --threads %u\n\n",
                    ac_version(), dir.c_str(), min_identity, max_unitigs, mad, threads);
        // check_settings, trim.rs:56-67 (misc.rs:98-119)
        int rc;
        if ((rc = check_dir(dir)) != AC_OK || (rc = dirs.add(dir)) != AC_OK || (rc = check_file(in_gfa)) != AC_OK) return rc;
        if (!(min_identity >= 0.0 && min_identity <= 1.0)) return set_error(nullptr, AC_EINPUT, "--min_identity must be between 0.0 and 1 (inclusive)");
        if (threads < 1) return set_error(nullptr, AC_EINPUT, "--threads cannot be less than 1");
        if (threads > 100) return set_error(nullptr, AC_EINPUT, "--threads cannot be greater than 100");
        if (mad < 0.0) return set_error(nullptr, AC_EINPUT, "--mad cannot be less than 0");
        std::string text;
        if ((rc = read_file(in_gfa, text)) != AC_OK || (!h && (rc = make_handle(device, h)) != AC_OK) || (rc = load_graph(text, graphs[i], seqs[i])) != AC_OK) return rc;
        if ((verbose & AC_VERBOSE_REPORT) && max_unitigs == 0) fprintf(log, "Since --max_unitigs was set to 0, trimming is disabled.\n\n");
    }
    std::vector<TrimCluster> clusters;
    for (uint32_t i = 0; i < n; ++i) clusters.push_back(TrimCluster{&graphs[i], &seqs[i], (verbose & AC_VERBOSE_REPORT) ? reports[i] : nullptr, TrimStats()});
    AlignBatch batch;
    trim_graphs(h->align_device(), clusters, min_identity, max_unitigs, mad, batch);
    std::vector<std::string> gfa(n), yaml(n);
    for (uint32_t i = 0; i < n; ++i) { graphs[i].gfa_text(seqs[i], gfa[i]); yaml[i] = trimmed_metrics_yaml(seqs[i]); }
    for (uint32_t i = 0; i < n; ++i) {
        const std::string dir = cluster_dirs[i], out_gfa = dir + "/2_trimmed.gfa", out_yaml = dir + "/2_trimmed.yaml";
        if (!write_file(out_gfa, gfa[i])) return set_error(nullptr, AC_EIO, "cannot write " + out_gfa);
        if (!write_file(out_yaml, yaml[i])) return set_error(nullptr, AC_EIO, "cannot write " + out_yaml);
        const TrimStats& ts = clusters[i].stats;
        if (!(verbose & AC_VERBOSE_REPORT)) continue;
        if (n == 1) fprintf(reports[i], "\nFinished!\nUnitig graph of trimmed sequences: %s\n(%llu alignments, %llu DP cells, alignment kernels %.2f ms)\n\n", out_gfa.c_str(),
                            (unsigned long long)ts.jobs, (unsigned long long)ts.cells, (double)ts.kernel_ms);
        else fprintf(reports[i], "\nFinished!\nUnitig graph of trimmed sequences: %s\n(%llu alignments, %llu DP cells)\n\n", out_gfa.c_str(),
                     (unsigned long long)ts.jobs, (unsigned long long)ts.cells);
    }
    if (verbose && n > 1)
        fprintf(reports[n - 1], "Trimmed %u clusters: %u kernel launches, %llu alignments, %llu DP cells, alignment kernels %.2f ms\n", batch.clusters, batch.launches,
                (unsigned long long)batch.jobs, (unsigned long long)batch.cells, (double)batch.kernel_ms);
    fill_batch_info(batch, info);
    return ok(h.get());
    AC_GUARD_END(nullptr)
}

// resolve.rs:31-75 for n directories; ac_resolve_dir is n = 1
int resolve_dirs(const char* const* cluster_dirs, uint32_t n, int32_t verbose, int32_t device, ac_batch_info* info) {
    if (!cluster_dirs || n == 0) return set_error(nullptr, AC_EINVAL, n == 0 ? "no cluster directory" : "null argument");
    for (uint32_t i = 0; i < n; ++i) if (!cluster_dirs[i]) return set_error(nullptr, AC_EINVAL, "null argument");
    if (info) *info = ac_batch_info{};
    AC_GUARD_BEGIN
    DirReports reports(n);
    DirSet dirs;
    std::vector<std::string> texts(n);
    Handle h;
    for (uint32_t i = 0; i < n; ++i) {
        FILE* log = reports[i];
        const std::string dir = cluster_dirs[i], trimmed = dir + "/2_trimmed.gfa";
        if (verbose & AC_VERBOSE_BANNER) fprintf(log, "\nStarting autocycler resolve (%s)\n\n", ac_version());
        // check_settings, resolve.rs:72-75 (misc.rs:98-119)
        int rc;
        if ((rc = check_dir(dir)) != AC_OK || (rc = dirs.add(dir)) != AC_OK || (rc = check_file(trimmed)) != AC_OK) return rc;
        if ((rc = read_file(trimmed, texts[i])) != AC_OK || (!h && (rc = make_handle(device, h)) != AC_OK)) return rc;
        if (verbose & AC_VERBOSE_REPORT)
            fprintf(log, "\nStarting autocycler resolve\n    This command resolves repeats in the unitig graph.\n\nSettings:\n  --cluster_dir %s\n\n", dir.c_str());
        HostGraph g; std::vector<HostSeq> seqs;
        if ((rc = load_graph(texts[i], g, seqs)) != AC_OK) return rc;
    }
    std::vector<ResolveCluster> clusters;      // the files' own texts, as the reference re-reads them (resolve.rs:59)
    for (uint32_t i = 0; i < n; ++i) clusters.push_back(ResolveCluster{&texts[i], (verbose & AC_VERBOSE_REPORT) ? reports[i] : nullptr, {}, {}});
    AlignBatch batch;
    resolve_texts(h->align_device(), clusters, batch);
    for (uint32_t i = 0; i < n; ++i) {
        const std::string dir = cluster_dirs[i], bridged = dir + "/3_bridged.gfa", merged = dir + "/4_merged.gfa", final_gfa = dir + "/5_final.gfa";
        const ResolveResult& r = clusters[i].out;
        if (!write_file(bridged, r.bridged) || !write_file(merged, r.merged) || !write_file(final_gfa, r.final_gfa))
            return set_error(nullptr, AC_EIO, "cannot write the output files under " + dir);
        const ResolveStats& rs = clusters[i].stats;
        if (!(verbose & AC_VERBOSE_REPORT)) continue;
        if (n == 1) fprintf(reports[i], "\nFinished!\nFinal consensus graph: %s\n(%llu distance jobs, %llu DP cells, distance kernels %.2f ms)\n\n", final_gfa.c_str(),
                            (unsigned long long)rs.jobs, (unsigned long long)rs.cells, (double)rs.kernel_ms);
        else fprintf(reports[i], "\nFinished!\nFinal consensus graph: %s\n(%llu distance jobs, %llu DP cells)\n\n", final_gfa.c_str(),
                     (unsigned long long)rs.jobs, (unsigned long long)rs.cells);
    }
    if (verbose && n > 1)
        fprintf(reports[n - 1], "Resolved %u clusters: %u kernel launches, %llu distance jobs, %llu DP cells, distance kernels %.2f ms\n", batch.clusters, batch.launches,
                (unsigned long long)batch.jobs, (unsigned long long)batch.cells, (double)batch.kernel_ms);
    fill_batch_info(batch, info);
    return ok(h.get());
    AC_GUARD_END(nullptr)
}
}  // namespace

// trim.rs:288-326 for a batch of caller paths, one device round of overlap alignments
int ac_trim_paths(ac_handle* h, int32_t mode, const int32_t* paths, const uint64_t* path_off, uint64_t n_paths,
                  const uint32_t* weights, uint64_t n_weights, double min_identity, uint32_t max_unitigs,
                  int32_t* out, uint64_t* out_off, uint8_t* trimmed) {
    if (!h || !path_off || !weights || !out_off || !trimmed || (n_paths && path_off[n_paths] && (!paths || !out))) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    if (mode != AC_TRIM_START_END && mode != AC_TRIM_HAIRPIN_START && mode != AC_TRIM_HAIRPIN_END) return set_error(h, AC_EINVAL, "unknown trim mode");
    std::vector<std::vector<int32_t>> in(n_paths), res;
    for (uint64_t x = 0; x < n_paths; ++x) {
        const int rc = check_path(h, paths, path_off, x, n_weights);
        if (rc != AC_OK) return rc;
        in[x].assign(paths + path_off[x], paths + path_off[x + 1]);
    }
    std::vector<uint32_t> w(weights, weights + n_weights);
    std::vector<uint8_t> ok_flags;
    TrimStats st;
    trim_paths(h->align_device(), (TrimMode)mode, in, w, min_identity, max_unitigs, ok_flags, res, st);
    uint64_t at = 0;
    out_off[0] = 0;
    for (uint64_t x = 0; x < n_paths; ++x) {
        trimmed[x] = ok_flags[x];
        if (ok_flags[x]) { std::copy(res[x].begin(), res[x].end(), out + at); at += res[x].size(); }
        out_off[x + 1] = at;
    }
    h->t.trim_kernel = st.kernel_ms; h->trim_stats = st;
    return ok(h);
    AC_GUARD_END(h)
}

int ac_trim(ac_handle* h, double min_identity, uint32_t max_unitigs, double mad) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    AC_GUARD_BEGIN
    if (!h->built) return set_error(h, AC_EINVAL, "a graph must be built or loaded before ac_trim");
    ensure_graph(h);
    TrimStats st;
    trim_graph(h->graph, h->seqs, h->align_device(), min_identity, max_unitigs, mad, false, st);
    h->infos.clear(); h->ascii.clear();      // the sequences are trimmed paths now: no bytes
    h->trim_yaml = trimmed_metrics_yaml(h->seqs); h->trimmed = true;
    h->t.trim_kernel = st.kernel_ms; h->trim_stats = st;
    h->gfa_ready = false;
    return ok(h);
    AC_GUARD_END(h)
}

int ac_trim_yaml(ac_handle* h, char* out, uint64_t cap, uint64_t* length) {
    if (!h || !length) return set_error(h, AC_EINVAL, "null argument");
    if (!h->trimmed) return set_error(h, AC_EINVAL, "ac_trim must precede ac_trim_yaml");
    return copy_text(h, h->trim_yaml, out, cap, length);
}

int ac_trim_stats(const ac_handle* h, uint64_t* jobs, uint64_t* cells, uint32_t* max_window, uint64_t* max_path) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    if (jobs) *jobs = h->trim_stats.jobs;
    if (cells) *cells = h->trim_stats.cells;
    if (max_window) *max_window = h->trim_stats.max_window;
    if (max_path) *max_path = h->trim_stats.max_path;
    return ok(h);
}

int ac_trim_dir(const char* cluster_dir, double min_identity, uint32_t max_unitigs, double mad, uint32_t threads, int32_t device, int32_t verbose) {
    if (!cluster_dir) return set_error(nullptr, AC_EINVAL, "null argument");
    return trim_dirs(&cluster_dir, 1, min_identity, max_unitigs, mad, threads, device, verbose ? AC_VERBOSE_REPORT : 0, nullptr);
}

int ac_trim_dirs(const char* const* cluster_dirs, uint32_t n, double min_identity, uint32_t max_unitigs, double mad, uint32_t threads,
                 int32_t device, int32_t verbose, ac_batch_info* info) {
    return trim_dirs(cluster_dirs, n, min_identity, max_unitigs, mad, threads, device, verbose, info);
}

// UPGMA (cluster.rs:395-480) on a caller's symmetric matrix: the kernel that ac_cluster runs on the distances it leaves on the device
int ac_upgma(ac_handle* h, const double* sym_dist, uint32_t n, const uint32_t* ids, uint32_t* node, uint32_t* left, uint32_t* right, double* dist) {
    if (!h || (n && (!sym_dist || !ids)) || (n > 1 && (!node || !left || !right || !dist))) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    for (uint64_t i = 0; i < n; ++i)          // a NaN distance can leave no pair to merge (the reference panics there)
        for (uint64_t j = 0; j < n; ++j)
            if (i != j && sym_dist[i * n + j] != sym_dist[i * n + j]) return set_error(h, AC_EINPUT, "the distance matrix holds a NaN off its diagonal");
    std::vector<UpgmaMerge> m(n > 1 ? n - 1 : 0);
    h->cluster_stats.upgma_ms = h->cluster_device().upgma(sym_dist, n, ids, m.data());
    for (size_t x = 0; x < m.size(); ++x) { node[x] = m[x].node; left[x] = m[x].left; right[x] = m[x].right; dist[x] = m[x].dist; }
    return ok(h);
    AC_GUARD_END(h)
}

int ac_cluster(ac_handle* h, double cutoff, int64_t min_assemblies, const uint16_t* manual, uint64_t n_manual) {
    if (!h || (n_manual && !manual)) return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    if (!h->built) return set_error(h, AC_EINVAL, "a graph must be built or loaded before ac_cluster");
    if (cutoff <= 0.0 || cutoff >= 1.0) return set_error(h, AC_EINPUT, "--cutoff must be between 0 and 1 (exclusive)");
    if (min_assemblies == 0) return set_error(h, AC_EINPUT, "--min_assemblies must be 1 or greater");
    std::vector<uint16_t> man(manual, manual + n_manual);
    std::sort(man.begin(), man.end());
    ensure_graph(h);
    h->clustered = false;
    // the per-cluster graphs re-load the handle's graph as text, as the reference re-loads input_assemblies.gfa; the cluster numbers go
    // to a copy of the sequences, so the handle's own GFA output is unchanged
    std::string text;
    h->graph.gfa_text(h->seqs, text);
    std::vector<HostSeq> seqs = h->seqs;
    cluster_graph(text, h->graph, seqs, h->cluster_device(), cutoff, min_assemblies < 0 ? -1 : min_assemblies, man, 0xFFFFFFFFu, "clustering", false, h->cluster, h->cluster_stats);
    h->clustered = true;
    return ok(h);
    AC_GUARD_END(h)
}

int ac_cluster_text(ac_handle* h, int32_t what, uint32_t cluster, char* out, uint64_t cap, uint64_t* length) {
    if (!h || !length) return set_error(h, AC_EINVAL, "null argument");
    if (!h->clustered) return set_error(h, AC_EINVAL, "ac_cluster must precede ac_cluster_text");
    const ClusterResult& r = h->cluster;
    const bool per_cluster = what == AC_CLUSTER_GFA || what == AC_CLUSTER_UNTRIMMED_YAML;
    if (per_cluster && (cluster < 1 || cluster > r.cluster_gfa.size())) return set_error(h, AC_ERANGE, "no cluster " + std::to_string(cluster));
    const std::string* t = what == AC_CLUSTER_PHYLIP ? &r.phylip : what == AC_CLUSTER_NEWICK ? &r.newick : what == AC_CLUSTER_TSV ? &r.tsv :
                           what == AC_CLUSTER_YAML ? &r.yaml : what == AC_CLUSTER_GFA ? &r.cluster_gfa[cluster - 1] :
                           what == AC_CLUSTER_UNTRIMMED_YAML ? &r.cluster_yaml[cluster - 1] : nullptr;
    if (!t) return set_error(h, AC_EINVAL, "unknown cluster text");
    return copy_text(h, *t, out, cap, length);
}

int ac_cluster_assignments(const ac_handle* h, uint16_t* cluster, uint8_t* pass, uint64_t cap) {
    if (!h || !cluster || !pass) return set_error(h, AC_EINVAL, "null argument");
    if (!h->clustered) return set_error(h, AC_EINVAL, "ac_cluster must precede ac_cluster_assignments");
    const ClusterResult& r = h->cluster;
    if (cap < r.seq_cluster.size()) return set_error(h, AC_ERANGE, "buffer too small");
    for (size_t i = 0; i < r.seq_cluster.size(); ++i) { cluster[i] = r.seq_cluster[i]; pass[i] = r.cluster_pass[r.seq_cluster[i] - 1]; }
    return ok(h);
}

int ac_cluster_stats(const ac_handle* h, uint32_t* n_seqs, uint32_t* pass_clusters, uint32_t* fail_clusters, float* distance_ms, float* upgma_ms, double* cluster_gfa_ms) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    const ClusterStats& s = h->cluster_stats;
    if (n_seqs) *n_seqs = s.n_seqs;
    if (pass_clusters) *pass_clusters = s.pass_clusters;
    if (fail_clusters) *fail_clusters = s.fail_clusters;
    if (distance_ms) *distance_ms = s.distance_ms;
    if (upgma_ms) *upgma_ms = s.upgma_ms;
    if (cluster_gfa_ms) *cluster_gfa_ms = s.cluster_gfa_ms;
    return ok(h);
}

int ac_cluster_dir(const char* autocycler_dir, double cutoff, int64_t min_assemblies, uint32_t max_contigs, const char* manual, int32_t device, int32_t verbose) {
    if (!autocycler_dir) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    // check_settings (cluster.rs:67-76)
    const std::string dir = autocycler_dir, gfa = dir + "/input_assemblies.gfa", cdir = dir + "/clustering";
    int rc;
    if ((rc = check_dir(dir)) != AC_OK || (rc = check_file(gfa)) != AC_OK) return rc;
    if (cutoff <= 0.0 || cutoff >= 1.0) return set_error(nullptr, AC_EINPUT, "--cutoff must be between 0 and 1 (exclusive)");
    if (min_assemblies == 0) return set_error(nullptr, AC_EINPUT, "--min_assemblies must be 1 or greater");
    // delete_dir_if_exists (misc.rs:41-48): only a directory (or a link to one, which goes itself) is removed; anything else makes
    // create_dir fail below
    struct stat st;
    if (stat(cdir.c_str(), &st) == 0 && S_ISDIR(st.st_mode)) {
        struct stat lst;
        const int removed = lstat(cdir.c_str(), &lst) == 0 && S_ISLNK(lst.st_mode) ? unlink(cdir.c_str()) : remove_tree(cdir);
        if (removed != 0) return set_error(nullptr, AC_EINPUT, "failed to delete directory " + cdir + "\n" + strerror(errno));
    }
    if (mkdir(cdir.c_str(), 0777) != 0) return set_error(nullptr, AC_EINPUT, "failed to create directory " + cdir + "\n" + strerror(errno));
    if (verbose) fprintf(stderr, "\nStarting autocycler cluster\n    This command takes a unitig graph (made by autocycler compress) and clusters the sequences based on "
                                 "their similarity. Ideally, each cluster will then contain sequences which can be combined into a consensus.\n\n");
    std::string text; Handle h;
    if ((rc = read_file(gfa, text)) != AC_OK || (rc = make_handle(device, h)) != AC_OK || (rc = load_input_gfa(h.get(), text)) != AC_OK) return rc;
    const std::vector<uint16_t> man = manual ? parse_manual_clusters(manual) : std::vector<uint16_t>();
    if (verbose) fprintf(stderr, "Settings:\n  --autocycler_dir %s\n", dir.c_str());
    cluster_graph(text, h->graph, h->seqs, h->cluster_device(), cutoff, min_assemblies < 0 ? -1 : min_assemblies, man, max_contigs, cdir, verbose != 0, h->cluster, h->cluster_stats);
    const ClusterResult& r = h->cluster;
    const std::string phylip = cdir + "/pairwise_distances.phylip", newick = cdir + "/clustering.newick", tsv = cdir + "/clustering.tsv";
    bool good = write_file(phylip, r.phylip) && write_file(newick, r.newick);
    for (size_t c = 0; good && c < r.cluster_gfa.size(); ++c) {
        char name[32]; snprintf(name, sizeof name, "/cluster_%03zu", c + 1);
        const std::string sub = cdir + (r.cluster_pass[c] ? "/qc_pass" : "/qc_fail"), cd = sub + name;
        mkdir(sub.c_str(), 0777);
        good = mkdir(cd.c_str(), 0777) == 0 && write_file(cd + "/1_untrimmed.gfa", r.cluster_gfa[c]) && write_file(cd + "/1_untrimmed.yaml", r.cluster_yaml[c]);
    }
    good = good && write_file(tsv, r.tsv) && write_file(cdir + "/clustering.yaml", r.yaml);
    if (!good) return set_error(nullptr, AC_EIO, "cannot write the output files under " + cdir);
    if (verbose) fprintf(stderr, "\nFinished!\n    You can now run autocycler trim on each cluster. If you want to manually inspect the clustering, you can "
                                 "view the following files.\nPairwise distances:         %s\nClustering tree (Newick):   %s\nClustering tree (metadata): %s\n"
                                 "\n(distance kernels %.2f ms, UPGMA kernel %.2f ms, per-cluster graphs %.1f ms)\n\n", phylip.c_str(), newick.c_str(), tsv.c_str(),
                         (double)h->cluster_stats.distance_ms, (double)h->cluster_stats.upgma_ms, h->cluster_stats.cluster_gfa_ms);
    return ok(h.get());
    AC_GUARD_END(nullptr)
}

// Bridge::new (resolve.rs:430-462) for caller groups of paths, one device round of distances
int ac_bridge_best_paths(ac_handle* h, const int32_t* paths, const uint64_t* path_off, uint64_t n_paths, const uint64_t* group_off, uint64_t n_groups,
                         const uint32_t* weights, uint64_t n_weights, uint32_t* totals, int32_t* best, uint64_t* best_off) {
    if (!h || !path_off || !group_off || !best_off || (n_weights && !weights) || (n_paths && !totals) || (n_paths && path_off[n_paths] && (!paths || !best)))
        return set_error(h, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    if (group_off[0] != 0 || group_off[n_groups] != n_paths) return set_error(h, AC_EINVAL, "the groups must cover the paths in order");
    std::vector<std::vector<std::vector<int32_t>>> groups(n_groups);
    for (uint64_t g = 0; g < n_groups; ++g) {
        if (group_off[g + 1] < group_off[g]) return set_error(h, AC_EINVAL, "group offsets must not decrease");
        for (uint64_t x = group_off[g]; x < group_off[g + 1]; ++x) {
            const int rc = check_path(h, paths, path_off, x, n_weights);
            if (rc != AC_OK) return rc;
            groups[g].emplace_back(paths + path_off[x], paths + path_off[x + 1]);
        }
    }
    std::vector<uint32_t> w(weights, weights + n_weights);
    std::vector<std::vector<uint32_t>> tot;
    std::vector<std::vector<int32_t>> bp;
    ResolveStats st;
    bridge_best_paths(h->align_device(), groups, w, tot, bp, st);
    uint64_t at = 0;
    best_off[0] = 0;
    for (uint64_t g = 0; g < n_groups; ++g) {
        std::copy(tot[g].begin(), tot[g].end(), totals + group_off[g]);
        std::copy(bp[g].begin(), bp[g].end(), best + at); at += bp[g].size();
        best_off[g + 1] = at;
    }
    h->resolve_stats = st;
    return ok(h);
    AC_GUARD_END(h)
}

int ac_resolve(ac_handle* h, int32_t verbose) {
    if (!h) return set_error(nullptr, AC_EINVAL, "null handle");
    AC_GUARD_BEGIN
    if (!h->built) return set_error(h, AC_EINVAL, "a graph must be loaded before ac_resolve");
    ensure_graph(h);
    h->resolved = false;
    std::string text;                      // the graph as a 2_trimmed.gfa: resolve re-loads it for its second pass (resolve.rs:59)
    h->graph.gfa_text(h->seqs, text);
    resolve_text(text, h->align_device(), verbose != 0, h->resolve, h->resolve_stats);
    h->resolved = true;
    return ok(h);
    AC_GUARD_END(h)
}

int ac_resolve_text(ac_handle* h, int32_t what, char* out, uint64_t cap, uint64_t* length) {
    if (!h || !length) return set_error(h, AC_EINVAL, "null argument");
    if (!h->resolved) return set_error(h, AC_EINVAL, "ac_resolve must precede ac_resolve_text");
    const std::string* t = what == AC_RESOLVE_BRIDGED ? &h->resolve.bridged : what == AC_RESOLVE_MERGED ? &h->resolve.merged :
                           what == AC_RESOLVE_FINAL ? &h->resolve.final_gfa : nullptr;
    if (!t) return set_error(h, AC_EINVAL, "unknown resolve text");
    return copy_text(h, *t, out, cap, length);
}

int ac_resolve_stats(const ac_handle* h, ac_resolve_info* out) {
    if (!h || !out) return set_error(h, AC_EINVAL, "null argument");
    const ResolveStats& s = h->resolve_stats;
    out->anchors = s.anchors; out->unique_bridges = s.unique_bridges; out->conflicting_bridges = s.conflicting_bridges; out->culled_bridges = s.culled_bridges;
    out->jobs = s.jobs; out->cells = s.cells; out->longest_path = s.longest_path; out->shared_jobs = s.shared_jobs; out->hbm_jobs = s.hbm_jobs;
    out->kernel_ms = s.kernel_ms;
    return ok(h);
}

int ac_resolve_dir(const char* cluster_dir, int32_t verbose, int32_t device) {
    if (!cluster_dir) return set_error(nullptr, AC_EINVAL, "null argument");
    return resolve_dirs(&cluster_dir, 1, verbose ? AC_VERBOSE_REPORT : 0, device, nullptr);
}

int ac_resolve_dirs(const char* const* cluster_dirs, uint32_t n, int32_t verbose, int32_t device, ac_batch_info* info) {
    return resolve_dirs(cluster_dirs, n, verbose, device, info);
}

int ac_combine_dir(const char* autocycler_dir, const char* const* in_gfas, uint32_t n_gfas, int32_t verbose) {
    if (!autocycler_dir || (n_gfas && !in_gfas)) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    if (n_gfas == 0) return set_error(nullptr, AC_EINPUT, "at least one input GFA is required");
    std::vector<std::string> names, texts(n_gfas);
    for (uint32_t i = 0; i < n_gfas; ++i) { if (!in_gfas[i]) return set_error(nullptr, AC_EINVAL, "null argument"); names.push_back(in_gfas[i]); }
    for (const std::string& n : names) if (check_file(n) != AC_OK) return AC_EINPUT;     // check_settings (combine.rs:52-56)
    const std::string dir = autocycler_dir;
    if (!make_dirs(dir)) return set_error(nullptr, AC_EINPUT, "failed to create directory " + dir + "\n" + strerror(errno));
    if (verbose) {
        fprintf(stderr, "\nStarting autocycler combine\n    This command combines different clusters into a single assembly file.\n\nSettings:\n  --autocycler_dir %s\n  --in_gfas %s\n",
                dir.c_str(), names[0].c_str());
        for (size_t i = 1; i < names.size(); ++i) fprintf(stderr, "            %s\n", names[i].c_str());
        fprintf(stderr, "\n");
    }
    for (uint32_t i = 0; i < n_gfas; ++i) if (read_file(names[i], texts[i]) != AC_OK) return AC_EIO;
    std::string gfa, fasta, yaml;
    combine_texts(texts, names, verbose != 0, gfa, fasta, yaml);
    const std::string out_gfa = dir + "/consensus_assembly.gfa", out_fasta = dir + "/consensus_assembly.fasta", out_yaml = dir + "/consensus_assembly.yaml";
    if (!write_file(out_gfa, gfa) || !write_file(out_fasta, fasta) || !write_file(out_yaml, yaml)) return set_error(nullptr, AC_EIO, "cannot write the output files under " + dir);
    if (verbose) fprintf(stderr, "\nFinished!\nCombined graph: %s\nCombined fasta: %s\n\n%s\n\n", out_gfa.c_str(), out_fasta.c_str(),
                         yaml.find("fully_resolved: true") != std::string::npos ? "Consensus assembly is fully resolved" : "One or more clusters failed to fully resolve");
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

// ---- `autocycler clean`, `autocycler gfa2fasta` and `autocycler table` (host only) ----------------------------------------------
int ac_clean_gfa(const char* in_gfa, const char* out_gfa, const char* remove, const char* duplicate, const double* min_depth, int32_t verbose) {
    if (!in_gfa || !out_gfa) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    const std::string in = in_gfa, out = out_gfa;
    int rc;
    if ((rc = check_file(in)) != AC_OK) return rc;        // check_settings (clean.rs:47-49)
    if (verbose) fprintf(stderr, "\nStarting autocycler clean\n    This command removes user-specified tigs from a combined Autocycler graph and then merges "
                                 "all linear paths to produce a clean output graph.\n\n");
    const std::vector<uint32_t> rm = remove ? parse_tig_numbers(remove) : std::vector<uint32_t>(),
                                dup = duplicate ? parse_tig_numbers(duplicate) : std::vector<uint32_t>();
    auto joined = [](const std::vector<uint32_t>& v) { std::string s; for (uint32_t n : v) s += (s.empty() ? "" : ",") + std::to_string(n); return s; };
    if (verbose) {
        fprintf(stderr, "Settings:\n  --in_gfa %s\n  --out_gfa %s\n", in.c_str(), out.c_str());
        if (!rm.empty()) fprintf(stderr, "  --remove %s\n", joined(rm).c_str());
        if (!dup.empty()) fprintf(stderr, "  --duplicate %s\n", joined(dup).c_str());
        fprintf(stderr, "\n\nLoading graph\n    The unitig graph is now loaded into memory.\n\n");
    }
    std::string text, gfa;
    if ((rc = read_file(in, text)) != AC_OK) return rc;
    HostGraph g;
    load_user_gfa(text, g);
    if (verbose) fprintf(stderr, "%u unitig%s, %llu link%s\ntotal length: %llu bp\n\n", g.U, g.U == 1 ? "" : "s", (unsigned long long)g.link_count_single(),
                         g.link_count_single() == 1 ? "" : "s", (unsigned long long)g.total_length());
    clean_graph(g, in, rm, dup, min_depth, true, verbose != 0, gfa);
    if (!write_file(out, gfa)) return set_error(nullptr, AC_EIO, "cannot write " + out);
    if (verbose) fprintf(stderr, "\nFinished!\nCleaned graph: %s\n\n", out.c_str());
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

int ac_clean_text(const char* gfa_text, uint64_t length, const uint32_t* remove, uint64_t n_remove, const uint32_t* duplicate, uint64_t n_duplicate,
                  const double* min_depth, int32_t merge, char* out, uint64_t cap, uint64_t* out_length) {
    if (!gfa_text || !out_length || (n_remove && !remove) || (n_duplicate && !duplicate)) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    HostGraph g;
    load_user_gfa(std::string(gfa_text, length), g);
    std::string gfa;
    clean_graph(g, "the GFA", std::vector<uint32_t>(remove, remove + n_remove), std::vector<uint32_t>(duplicate, duplicate + n_duplicate),
                min_depth, merge != 0, false, gfa);
    return copy_text(nullptr, gfa, out, cap, out_length);
    AC_GUARD_END(nullptr)
}

int ac_gfa_to_fasta(const char* in_gfa, const char* out_fasta, int32_t verbose) {
    if (!in_gfa || !out_fasta) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    const std::string in = in_gfa, out = out_fasta;
    int rc;
    if ((rc = check_file(in)) != AC_OK) return rc;
    if (verbose) fprintf(stderr, "\nStarting autocycler gfa2fasta\n    This command loads an Autocycler graph and saves it as a FASTA file with topological "
                                 "information in the sequence headers.\n\nSettings:\n  --in_gfa %s\n  --out_fasta %s\n\n\nLoading graph\n    The unitig graph "
                                 "is now loaded into memory.\n\n", in.c_str(), out.c_str());
    std::string text;
    if ((rc = read_file(in, text)) != AC_OK) return rc;
    HostGraph g;
    load_user_gfa(text, g);
    if (verbose) fprintf(stderr, "%u unitig%s, %llu link%s\ntotal length: %llu bp\n\n\nSaving to FASTA\n    The unitig graph is now saved to a FASTA file.\n\n",
                         g.U, g.U == 1 ? "" : "s", (unsigned long long)g.link_count_single(), g.link_count_single() == 1 ? "" : "s",
                         (unsigned long long)g.total_length());
    uint64_t counts[3];
    const std::string fasta = gfa_fasta_text(g, counts);
    if (!write_file(out, fasta)) return set_error(nullptr, AC_EIO, "cannot write " + out);
    if (verbose) {
        const char* what[3] = {"circular", "linear", "other"};
        for (int i = 0; i < 3; ++i) fprintf(stderr, "%llu %s sequence%s\n", (unsigned long long)counts[i], what[i], counts[i] == 1 ? "" : "s");
        fprintf(stderr, "\n");
    }
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

int ac_gfa_fasta_text(const char* gfa_text, uint64_t length, char* out, uint64_t cap, uint64_t* out_length) {
    if (!gfa_text || !out_length) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    HostGraph g;
    load_user_gfa(std::string(gfa_text, length), g);
    uint64_t counts[3];
    return copy_text(nullptr, gfa_fasta_text(g, counts), out, cap, out_length);
    AC_GUARD_END(nullptr)
}

int ac_table_text(const char* autocycler_dir, const char* name, const char* fields, uint64_t sigfigs, int32_t verbose, char* out, uint64_t cap,
                  uint64_t* length) {
    if (!length) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    int rc;
    if (autocycler_dir && (rc = check_dir(autocycler_dir)) != AC_OK) return rc;     // check_settings (table.rs:34-41)
    const std::string line = table_text(autocycler_dir ? autocycler_dir : "", autocycler_dir != nullptr, name ? name : "",
                                        fields ? fields : TABLE_DEFAULT_FIELDS, sigfigs, verbose != 0);
    return copy_text(nullptr, line, out, cap, length);
    AC_GUARD_END(nullptr)
}

// ---- `autocycler dotplot` (dotplot.rs) ------------------------------------------------------------------------------------------
namespace {
// One dotplot device object per device, on a stream of its own, kept for the process so that its device buffers are reused by the next
// call.  The lock is held for the whole call: calls on one device run one at a time.
std::mutex g_dotplot_mu;
struct DotplotDevice {
    DeviceContext ctx; DeviceDotplot plot;
    explicit DotplotDevice(int32_t device) : ctx(device, nullptr), plot(ctx) {}
};
DeviceDotplot& dotplot_device(int32_t device) {           // with g_dotplot_mu held
    static std::vector<std::pair<int32_t, DotplotDevice*>> devices;
    for (auto& d : devices) if (d.first == device) return d.second->plot;
    devices.emplace_back(device, new DotplotDevice(device));
    return devices.back().second->plot;
}
void fill_info(const DotplotStats& st, ac_dotplot_info* info) {
    if (!info) return;
    info->windows = st.windows; info->groups = st.groups; info->dots = st.dots; info->host_windows = st.host_windows;
    info->bp_per_pixel = st.bp_per_pixel; info->text_height = st.text_height; info->kernel_ms = st.kernel_ms;
}
// font: a TrueType file, "" for no labels, NULL for the first standard DejaVuSans.ttf that exists (none: no labels, and a warning)
std::shared_ptr<DotplotFont> dotplot_font(const char* font, bool warn) {
    if (font && *font) return dotplot_font_load(font);
    if (font) return nullptr;
    std::shared_ptr<DotplotFont> f = dotplot_font_default(nullptr);
    if (!f && warn) fprintf(stderr, "Warning: no font found (DejaVuSans.ttf; give one with --font), so the sequence labels are not drawn\n");
    return f;
}
}  // namespace

int ac_dotplot_rgb(const char* const* seqs, const uint64_t* lengths, const char* const* filenames, const char* const* names, uint32_t n,
                   uint32_t res, uint32_t kmer, const char* font, int32_t device, uint8_t* rgb, ac_dotplot_info* info) {
    if ((n && (!seqs || !lengths || !names)) || !rgb) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    dotplot_check_settings(res, kmer);
    std::vector<DotplotInput> in(n);
    for (uint32_t i = 0; i < n; ++i) {
        if ((lengths[i] && !seqs[i]) || !names[i]) return set_error(nullptr, AC_EINVAL, "null argument");
        in[i].filename = filenames && filenames[i] ? filenames[i] : "";
        in[i].name = names[i];
        in[i].seq.assign(seqs[i] ? seqs[i] : "", lengths[i]);
        for (char& c : in[i].seq) if (c >= 'a' && c <= 'z') c = (char)(c - 32);
    }
    if (n == 0) return set_error(nullptr, AC_EINPUT, "no sequences were loaded");
    std::set<std::pair<std::string, std::string>> seen;
    for (const DotplotInput& d : in) if (!seen.insert({d.filename, d.name}).second) return set_error(nullptr, AC_EINPUT, "two sequences are named " + (d.filename.empty() ? d.name : d.filename + " " + d.name));
    const std::shared_ptr<DotplotFont> f = dotplot_font(font, false);
    std::vector<uint8_t> img;
    DotplotStats st;
    {
        std::lock_guard<std::mutex> lock(g_dotplot_mu);
        dotplot_image(dotplot_device(device), in, res, kmer, f.get(), img, st);
    }
    memcpy(rgb, img.data(), img.size());
    fill_info(st, info);
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

int ac_dotplot_dir(const char* input, const char* out_png, uint32_t res, uint32_t kmer, const char* font, int32_t device, int32_t verbose,
                   ac_dotplot_info* info) {
    if (!input || !out_png) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    dotplot_check_settings(res, kmer);                                                  // dotplot.rs:44-52
    const std::vector<DotplotInput> seqs = dotplot_load(input, verbose != 0);
    const std::shared_ptr<DotplotFont> f = dotplot_font(font, true);
    if (verbose) fprintf(stderr, "Creating dotplot\n    K-mers common between sequences are now used to build the dotplot image.\n\n");
    std::vector<uint8_t> img;
    DotplotStats st;
    {
        std::lock_guard<std::mutex> lock(g_dotplot_mu);
        dotplot_image(dotplot_device(device), seqs, res, kmer, f.get(), img, st);
    }
    if (!png_write(out_png, img.data(), res, res)) return set_error(nullptr, AC_EIO, std::string("cannot write ") + out_png);
    fill_info(st, info);
    if (verbose) {
        const uint64_t count = (uint64_t)seqs.size() * seqs.size();
        fprintf(stderr, "%llu pairwise dotplot%s drawn to image\n\nFinished!\nPairwise dotplots: %s\n(%llu windows, %llu dots, kernels %.2f ms)\n\n",
                (unsigned long long)count, count == 1 ? "" : "s", out_png, (unsigned long long)st.windows, (unsigned long long)st.dots, (double)st.kernel_ms);
    }
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

int ac_png_write(const char* path, const uint8_t* rgb, uint32_t width, uint32_t height) {
    if (!path || !rgb) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    if (!png_write(path, rgb, width, height)) return set_error(nullptr, AC_EIO, std::string("cannot write ") + path);
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

// ---- `autocycler subsample` (subsample.rs) --------------------------------------------------------------------------------------
namespace {
// One subsample device object per device, as for dotplot: its buffers (and pinned windows) are kept for the next call on that device.
// genome_size, depth, qv, unassembled, polish and variants read through the same object and keep their packed streams and tables beside it.
std::mutex g_subsample_mu;
struct SubsampleDevice {
    DeviceContext ctx; DeviceSubsample sub; DeviceSpectrum spec; DeviceDepth depth; DeviceQv qv; DeviceUnassembled unassembled; DevicePolish polish;
    DeviceVariants variants;
    explicit SubsampleDevice(int32_t device)
        : ctx(device, nullptr), sub(ctx), spec(ctx), depth(ctx), qv(ctx), unassembled(ctx), polish(ctx), variants(ctx) {}
};
SubsampleDevice& subsample_device(int32_t device) {        // with g_subsample_mu held
    static std::vector<std::pair<int32_t, SubsampleDevice*>> devices;
    for (auto& d : devices) if (d.first == device) return *d.second;
    devices.emplace_back(device, new SubsampleDevice(device));
    return *devices.back().second;
}
}  // namespace

int ac_subsample_dir(const char* reads, const char* out_dir, const char* genome_size, uint64_t count, double min_read_depth, uint64_t seed,
                     int32_t device, int32_t verbose, ac_subsample_info* info) {
    if (!reads || !out_dir || !genome_size) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    const std::string in = reads, dir = out_dir;
    const uint64_t gsize = parse_genome_size(genome_size);                    // subsample.rs:31-33, then check_settings (:47-55)
    int rc;
    if ((rc = check_file(in)) != AC_OK) return rc;
    struct stat st;
    if (stat(dir.c_str(), &st) == 0 && !S_ISDIR(st.st_mode)) return set_error(nullptr, AC_EINPUT, dir + " exists but is not a directory");
    if (gsize < 1) return set_error(nullptr, AC_EINPUT, "--genome_size must be at least 1");
    if (count < 2) return set_error(nullptr, AC_EINPUT, "--count must be at least 2");
    if (min_read_depth <= 0.0) return set_error(nullptr, AC_EINPUT, "--min_read_depth must be greater than 0");
    if (!make_dirs(dir)) return set_error(nullptr, AC_EINPUT, "failed to create directory " + dir + "\n" + strerror(errno));
    if (verbose) fprintf(stderr, "\nStarting autocycler subsample\n    This command subsamples a long-read set into subsets that are maximally independent "
                                 "from each other.\n\nSettings:\n  --reads %s\n  --out_dir %s\n  --genome_size %llu\n  --count %llu\n  --min_read_depth %s\n"
                                 "  --seed %llu\n\n", in.c_str(), dir.c_str(), (unsigned long long)gsize, (unsigned long long)count,
                         format_float(min_read_depth).c_str(), (unsigned long long)seed);
    SubsampleRun run;
    try {
        std::lock_guard<std::mutex> lock(g_subsample_mu);
        subsample_run(subsample_device(device).sub, in, dir, gsize, count, min_read_depth, seed, subsample_window_size(), verbose != 0, run);
    } catch (const AcIoError& e) { return set_error(nullptr, AC_EIO, e.msg); }
    catch (const std::length_error& e) { return set_error(nullptr, AC_ERANGE, e.what()); }
    if (info) {
        info->genome_size = run.genome_size; info->reads_per_subset = run.reads_per_subset;
        info->input_count = run.input.count; info->input_bases = run.input.bases; info->input_n50 = run.input.n50;
        info->windows = run.windows; info->bytes_scanned = run.bytes_scanned; info->kernel_ms = run.kernel_ms;
        info->read_ms = run.read_ms; info->shuffle_ms = run.shuffle_ms; info->write_ms = run.write_ms; info->copy_ms = run.copy_ms;
    }
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

int ac_subsample_words(uint64_t seed, uint32_t rounds, uint32_t* out, uint64_t n) {
    if (!out && n) return set_error(nullptr, AC_EINVAL, "null argument");
    if (rounds != 12 && rounds != 20) return set_error(nullptr, AC_EINVAL, "rounds must be 12 or 20");
    AC_GUARD_BEGIN
    const std::vector<uint32_t> w = subsample_rng_words(seed, n, (int)rounds);
    if (n) memcpy(out, w.data(), n * 4);
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

int ac_subsample_shuffle(uint64_t n, uint64_t seed, uint32_t* order) {
    if (!order && n) return set_error(nullptr, AC_EINVAL, "null argument");
    if (n >= 0xFFFFFFFFull) return set_error(nullptr, AC_ERANGE, "2^32 - 1 reads or more");
    AC_GUARD_BEGIN
    const std::vector<uint32_t> o = subsample_shuffle(n, seed);
    if (n) memcpy(order, o.data(), n * 4);
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

int ac_genome_size(const char* text, uint64_t* size) {
    if (!text || !size) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    *size = parse_genome_size(text);
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

// ---- `autocycler helper genome_size`: a k-mer depth estimate in place of helper.rs:388-403's Raven assembly --------------------------
static_assert(AC_GENOME_SIZE_BINS == AC_GS_BINS, "the header's bin count is the device's");
namespace {
void fill_gs_info(const GenomeSizeRun& r, ac_genome_size_info* info) {
    if (!info) return;
    *info = ac_genome_size_info{};
    info->estimate = r.estimate; info->k = r.k; info->reruns = (uint32_t)r.spectrum.reruns;
    info->reads = r.reads; info->bases = r.bases; info->windows = r.windows; info->distinct = r.distinct;
    info->valley = r.valley; info->peak = r.peak; info->peak_refined = r.peak_refined; info->solid = r.solid;
    info->partitions = r.spectrum.partitions; info->table_bytes = r.spectrum.table_bytes;
    info->kernel_ms = r.kernel_ms; info->scan_ms = r.scan_ms; info->pack_ms = r.spectrum.pack_ms; info->count_ms = r.spectrum.count_ms;
    info->hist_ms = r.spectrum.hist_ms; info->read_ms = r.read_ms; info->copy_ms = r.copy_ms;
}
}  // namespace

int ac_genome_size_estimate(const char* reads, uint32_t k, int32_t device, const char* dir, int32_t verbose, uint64_t* hist,
                            ac_genome_size_info* info) {
    if (!reads) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    const std::string in = reads;
    int rc;
    if ((rc = check_file(in)) != AC_OK) return rc;
    if (k < 11 || k > 31 || k % 2 == 0) return set_error(nullptr, AC_EINPUT, "--kmer must be odd and between 11 and 31");
    struct stat st;
    if (dir && stat(dir, &st) == 0 && !S_ISDIR(st.st_mode)) return set_error(nullptr, AC_EINPUT, std::string(dir) + " exists but is not a directory");
    if (dir && !make_dirs(dir)) return set_error(nullptr, AC_EINPUT, std::string("failed to create directory ") + dir + "\n" + strerror(errno));
    if (verbose) fprintf(stderr, "\nStarting autocycler helper genome_size\n    This build estimates the genome size from the reads' k-mer depth "
                                 "spectrum on the GPU. The reference assembles the reads with Raven and reports the assembly's length "
                                 "instead, so the two numbers differ.\n\nSettings:\n  --reads %s\n  --kmer %u\n\n", in.c_str(), k);
    GenomeSizeRun run;
    std::vector<uint64_t> h;
    try {
        std::lock_guard<std::mutex> lock(g_subsample_mu);
        SubsampleDevice& d = subsample_device(device);
        genome_size_run(d.sub, d.spec, in, k, subsample_window_size(), h, run);
    } catch (const AcIoError& e) { return set_error(nullptr, AC_EIO, e.msg); }
    catch (const std::length_error& e) { return set_error(nullptr, AC_ERANGE, e.what()); }
    if (hist) memcpy(hist, h.data(), AC_GS_BINS * 8);
    if (dir) {
        std::string tsv;
        for (uint64_t c = 1; c < AC_GS_BINS; ++c)
            if (h[c]) tsv += std::to_string(c) + "\t" + std::to_string(h[c]) + "\n";
        const std::string path = std::string(dir) + "/kmer_histogram.tsv";
        if (!write_file(path, tsv)) return set_error(nullptr, AC_EIO, "cannot write " + path);
    }
    genome_size_rule(h.data(), run.windows, run);
    fill_gs_info(run, info);
    if (verbose) fprintf(stderr, "K-mer spectrum (k = %u):\n  reads: %llu\n  bases: %llu\n  k-mer windows: %llu\n  distinct k-mers: %llu\n"
                                 "  valley: %llu\n  peak: %llu (refined %.3f)\n  solid k-mer occurrences: %llu\n  partitions: %llu\n\n"
                                 "Estimated genome size: %llu bp\n\n", k, (unsigned long long)run.reads, (unsigned long long)run.bases,
                         (unsigned long long)run.windows, (unsigned long long)run.distinct, (unsigned long long)run.valley,
                         (unsigned long long)run.peak, run.peak_refined, (unsigned long long)run.solid,
                         (unsigned long long)run.spectrum.partitions, (unsigned long long)run.estimate);
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

int ac_genome_size_from_histogram(const uint64_t* hist, uint64_t windows, ac_genome_size_info* info) {
    if (!hist) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    GenomeSizeRun run;
    genome_size_rule(hist, windows, run);
    fill_gs_info(run, info);
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

// ---- `autocycler depth`: read-measured contig depth (not in the reference) and helper.rs:889-931's depth filter ----------------------
int ac_depth_fasta(const char* assembly, const char* reads, const char* out_fasta, const char* tsv, int32_t source_header, uint32_t k,
                   const double* min_abs, const double* min_rel, int32_t device, int32_t verbose, double* depths, uint64_t* unique,
                   uint64_t cap, ac_depth_info* info) {
    if (!assembly || !out_fasta) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    const std::string in = assembly, out = out_fasta;
    int rc;
    if ((rc = check_file(in)) != AC_OK) return rc;
    if (!source_header) {
        if (!reads) return set_error(nullptr, AC_EINPUT, "--reads is required with --source reads (or use --source header)");
        if ((rc = check_file(reads)) != AC_OK) return rc;
        if (k < 11 || k > 31 || k % 2 == 0) return set_error(nullptr, AC_EINPUT, "--kmer must be odd and between 11 and 31");
    }
    if (verbose) {
        fprintf(stderr, "\nStarting autocycler depth\n    %s\n\nSettings:\n  --assembly %s\n  --out_fasta %s\n  --source %s\n",
                source_header ? "This command applies the reference's helper depth filter to the depths the contig headers carry."
                              : "This command measures each contig's read depth from the reads' k-mers on the GPU (an addition that is "
                                "not in the reference), then applies the reference's helper depth filter.",
                in.c_str(), out.c_str(), source_header ? "header" : "reads");
        if (!source_header) fprintf(stderr, "  --reads %s\n  --kmer %u\n", reads, k);
        if (min_abs) fprintf(stderr, "  --min_depth_abs %s\n", rust_fixed(*min_abs, 3).c_str());
        if (min_rel) fprintf(stderr, "  --min_depth_rel %s\n", rust_fixed(*min_rel, 3).c_str());
        fprintf(stderr, "\n");
    }
    ac_depth_info di{};
    di.k = source_header ? 0 : k;
    std::vector<FastaRecord> recs;
    std::vector<double> depth;
    std::vector<char> has;
    std::vector<uint64_t> uniq;
    if (source_header) {                                   // copy_fasta (helper.rs:577-585), then depth_filter on the copy
        std::vector<FastaRecord> loaded = parse_fasta(read_fasta_bytes(in), in);
        size_t bases = 0;
        for (const FastaRecord& r : loaded) bases += r.seq.size();
        if (bases == 0) {
            unlink(out.c_str());
            if (info) *info = di;
            return ok(nullptr);
        }
        recs = load_fasta(in);
        depth.assign(recs.size(), NAN); has.assign(recs.size(), 0); uniq.assign(recs.size(), 0);
        for (size_t i = 0; i < recs.size(); ++i) has[i] = depth_from_header(recs[i].header, depth[i]);
    } else {
        DepthResult r;
        {
            std::lock_guard<std::mutex> lock(g_subsample_mu);
            SubsampleDevice& d = subsample_device(device);
            try {
                depth_run(d.sub, d.spec, d.depth, in, reads, k, subsample_window_size(), r);
            } catch (const AcIoError& e) { return set_error(nullptr, AC_EIO, e.msg); }
            catch (const std::length_error& e) { return set_error(nullptr, AC_ERANGE, e.what()); }
        }
        recs = std::move(r.recs); depth = r.depth; uniq = r.unique;
        has.assign(recs.size(), 0);
        for (size_t i = 0; i < recs.size(); ++i) {
            has[i] = uniq[i] != 0;
            if (has[i]) recs[i].header += " depth=" + rust_fixed(depth[i], 2);
        }
        di.unique_kmers = r.unique_total; di.assembly_windows = r.device.assembly_windows; di.reads = r.reads;
        di.read_windows = r.read_windows; di.read_bases = r.read_bases; di.table_bytes = r.device.table_bytes;
        di.kernel_ms = r.kernel_ms; di.scan_ms = r.scan_ms; di.pack_ms = r.pack_reads_ms; di.insert_ms = r.device.pack_ms + r.device.insert_ms;
        di.probe_ms = r.device.probe_ms; di.median_ms = r.device.median_ms; di.read_ms = r.read_ms; di.copy_ms = r.copy_ms;
        if (verbose) {
            fprintf(stderr, "Read depth (k = %u):\n  reads: %llu\n  read k-mer windows: %llu\n  assembly k-mer windows: %llu\n  unique k-mers: %llu\n",
                    k, (unsigned long long)r.reads, (unsigned long long)r.read_windows, (unsigned long long)r.device.assembly_windows,
                    (unsigned long long)r.unique_total);
            for (size_t i = 0; i < recs.size(); ++i)
                fprintf(stderr, "  %s: %s (%llu unique k-mers)\n", recs[i].name.c_str(), has[i] ? ("depth=" + rust_fixed(depth[i], 2)).c_str() : "no depth",
                        (unsigned long long)uniq[i]);
        }
    }
    di.contigs = recs.size();
    std::vector<char> keep;
    std::string report;
    di.filtered = depth_filter(recs, depth, has, min_abs, min_rel, keep, report) ? 1 : 0;
    if ((min_abs || min_rel) && !di.filtered && verbose)
        fprintf(stderr, "\nNote: not every contig has a depth, so the depth filter keeps every contig, as the reference does\n");
    if (verbose) fputs(report.c_str(), stderr);
    std::string text;
    for (size_t i = 0; i < recs.size(); ++i)
        if (keep[i]) { text += ">" + recs[i].header + "\n" + recs[i].seq + "\n"; ++di.kept; }
    if (di.kept == 0) unlink(out.c_str());
    else if (!write_file(out, text)) return set_error(nullptr, AC_EIO, "cannot write " + out);
    if (tsv) {
        std::string t;
        for (size_t i = 0; i < recs.size(); ++i)
            t += recs[i].name + "\t" + std::to_string(recs[i].seq.size()) + "\t" + std::to_string(uniq[i]) + "\t" + (has[i] ? rust_fixed(depth[i], 2) : std::string()) + "\n";
        if (!write_file(tsv, t)) return set_error(nullptr, AC_EIO, std::string("cannot write ") + tsv);
    }
    for (uint64_t i = 0; i < std::min<uint64_t>(cap, recs.size()); ++i) {
        if (depths) depths[i] = has[i] ? depth[i] : NAN;
        if (unique) unique[i] = uniq[i];
    }
    if (info) *info = di;
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

int ac_depth_filter_text(const char* fasta_text, uint64_t length, const double* min_abs, const double* min_rel, char* out, uint64_t cap,
                         uint64_t* out_length) {
    if ((!fasta_text && length) || !out_length) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    std::string report;
    const std::string kept = depth_filter_text(std::string(fasta_text ? fasta_text : "", length), "the FASTA text", min_abs, min_rel, report);
    return copy_text(nullptr, kept, out, cap, out_length);
    AC_GUARD_END(nullptr)
}

int ac_depth_from_header(const char* header, double* depth) {
    if (!header || !depth) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    if (!depth_from_header(header, *depth)) return set_error(nullptr, AC_EINPUT, "the header carries no depth");
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

// ---- `autocycler qv`: each assembly's k-mer QV and completeness against the reads (not in the reference) -----------------------------
int ac_qv_dir(const char* reads, const char* const* inputs, uint32_t n_inputs, const char* out_dir, uint32_t k, const uint32_t* min_count,
              int32_t device, int32_t verbose, uint64_t* kmers, uint64_t* unsupported, uint64_t* solid_found, uint64_t cap, ac_qv_info* info) {
    if (!reads || !out_dir || (!inputs && n_inputs)) return set_error(nullptr, AC_EINVAL, "null argument");
    for (uint32_t i = 0; i < n_inputs; ++i) if (!inputs[i]) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    const std::string in = reads, dir = out_dir;
    if (!n_inputs) return set_error(nullptr, AC_EINPUT, "no assemblies given");
    if (k < 11 || k > 31 || k % 2 == 0) return set_error(nullptr, AC_EINPUT, "--kmer must be odd and between 11 and 31");
    if (min_count && (*min_count < 1 || *min_count > AC_GS_BINS - 1))
        return set_error(nullptr, AC_EINPUT, "--min_count must be between 1 and " + std::to_string(AC_GS_BINS - 1));
    int rc;
    if ((rc = check_file(in)) != AC_OK) return rc;
    const std::vector<std::string> paths = qv_inputs(std::vector<std::string>(inputs, inputs + n_inputs));
    struct stat st;
    if (stat(dir.c_str(), &st) == 0 && !S_ISDIR(st.st_mode)) return set_error(nullptr, AC_EINPUT, dir + " exists but is not a directory");
    if (!make_dirs(dir)) return set_error(nullptr, AC_EINPUT, "failed to create directory " + dir + "\n" + strerror(errno));
    if (verbose) {
        fprintf(stderr, "\nStarting autocycler qv\n    This command measures each assembly's k-mer accuracy (QV) and completeness against the reads, "
                        "counted on the GPU. It is not in the reference.\n\nSettings:\n  --reads %s\n  --assemblies", in.c_str());
        for (const std::string& p : paths) fprintf(stderr, " %s", p.c_str());
        fprintf(stderr, "\n  --out_dir %s\n  --kmer %u\n", dir.c_str(), k);
        if (min_count) fprintf(stderr, "  --min_count %u\n", *min_count);
        fprintf(stderr, "\n");
    }
    QvResult r;
    {
        std::lock_guard<std::mutex> lock(g_subsample_mu);
        SubsampleDevice& d = subsample_device(device);
        try {
            qv_run(d.sub, d.spec, d.qv, paths, in, k, min_count, subsample_window_size(), r);
        } catch (const AcIoError& e) { return set_error(nullptr, AC_EIO, e.msg); }
        catch (const std::length_error& e) { return set_error(nullptr, AC_ERANGE, e.what()); }
    }
    for (const char* sub : {"/unsupported", "/spectra_cn"})
        if (!make_dirs(dir + sub)) return set_error(nullptr, AC_EIO, "failed to create directory " + dir + sub + "\n" + strerror(errno));
    std::vector<std::pair<std::string, std::string>> files{{"qv.tsv", qv_table(r, k)}, {"contig_qv.tsv", qv_contig_table(r, k)},
                                                           {"kmer_histogram.tsv", qv_histogram(r)}};
    for (size_t a = 0; a < r.assemblies.size(); ++a) {
        files.emplace_back("unsupported/" + std::to_string(a + 1) + ".bed", r.assemblies[a].bed);
        files.emplace_back("spectra_cn/" + std::to_string(a + 1) + ".tsv", r.assemblies[a].spectrum);
    }
    for (const auto& f : files)
        if (!write_file(dir + "/" + f.first, f.second)) return set_error(nullptr, AC_EIO, "cannot write " + dir + "/" + f.first);
    uint64_t contigs = 0;
    for (size_t a = 0; a < r.assemblies.size(); ++a) {
        const QvAssembly& as = r.assemblies[a];
        contigs += as.contigs.size();
        if (a < cap) {
            if (kmers) kmers[a] = as.kmers;
            if (unsupported) unsupported[a] = as.unsupported;
            if (solid_found) solid_found[a] = as.solid_found;
        }
    }
    if (verbose) {
        fprintf(stderr, "K-mer QV (k = %u):\n  reads: %llu\n  read k-mer windows: %llu\n  distinct read k-mers: %llu\n  valley: %s\n"
                        "  min_count: %llu%s\n  solid read k-mers: %llu\n  assembly k-mer windows: %llu\n\n", k, (unsigned long long)r.reads,
                (unsigned long long)r.read_windows, (unsigned long long)r.distinct, r.valley ? std::to_string(r.valley).c_str() : "none",
                (unsigned long long)r.min_count, min_count ? " (given)" : " (the valley)", (unsigned long long)r.solid,
                (unsigned long long)r.device.assembly_windows);
        for (const QvAssembly& as : r.assemblies) {
            fprintf(stderr, "  %s: QV %s, %llu of %llu k-mers unsupported", as.path.c_str(), qv_text(as.unsupported, as.kmers, k).c_str(),
                    (unsigned long long)as.unsupported, (unsigned long long)as.kmers);
            if (r.solid) fprintf(stderr, ", completeness %.2f%%", 100.0 * (double)as.solid_found / (double)r.solid);
            fprintf(stderr, "\n");
        }
        fprintf(stderr, "\nFinished!\nQV table: %s/qv.tsv\n\n", dir.c_str());
    }
    if (info) {
        *info = ac_qv_info{};
        info->assemblies = r.assemblies.size(); info->contigs = contigs; info->k = k; info->min_count = (uint32_t)r.min_count;
        info->valley = r.valley; info->reads = r.reads; info->read_windows = r.read_windows; info->read_bases = r.read_bases;
        info->distinct = r.distinct; info->solid_kmers = r.solid; info->assembly_windows = r.device.assembly_windows;
        info->table_bytes = r.device.table_bytes; info->spectrum_table_bytes = r.spectrum.table_bytes; info->partitions = r.spectrum.partitions;
        info->reruns = r.spectrum.reruns;
        info->kernel_ms = r.kernel_ms; info->scan_ms = r.scan_ms; info->pack_ms = r.pack_reads_ms;
        info->insert_ms = r.device.pack_ms + r.device.insert_ms; info->probe_ms = r.device.probe_ms;
        info->count_ms = r.spectrum.count_ms + r.spectrum.hist_ms; info->assembly_ms = r.device.assembly_ms;
        info->read_ms = r.read_ms; info->copy_ms = r.copy_ms;
    }
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

// ---- `autocycler unassembled`: the reads an assembly does not explain (not in the reference) --------------------------------------
int ac_unassembled_dir(const char* reads, const char* const* inputs, uint32_t n_inputs, const char* out_dir, uint32_t k, const uint32_t* min_count,
                       uint64_t min_solid, double min_fraction, int32_t device, int32_t verbose, ac_unassembled_info* info) {
    if (!reads || !out_dir || (!inputs && n_inputs)) return set_error(nullptr, AC_EINVAL, "null argument");
    for (uint32_t i = 0; i < n_inputs; ++i) if (!inputs[i]) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    const std::string in = reads, dir = out_dir;
    if (!n_inputs) return set_error(nullptr, AC_EINPUT, "no assemblies given");
    if (k < 11 || k > 31 || k % 2 == 0) return set_error(nullptr, AC_EINPUT, "--kmer must be odd and between 11 and 31");
    if (min_count && (*min_count < 1 || *min_count > AC_GS_BINS - 1))
        return set_error(nullptr, AC_EINPUT, "--min_count must be between 1 and " + std::to_string(AC_GS_BINS - 1));
    if (min_solid < 1) return set_error(nullptr, AC_EINPUT, "--min_solid must be at least 1");
    if (!(min_fraction > 0.0 && min_fraction <= 1.0)) return set_error(nullptr, AC_EINPUT, "--min_fraction must be above 0 and at most 1");
    int rc;
    if ((rc = check_file(in)) != AC_OK) return rc;
    const std::vector<std::string> paths = qv_inputs(std::vector<std::string>(inputs, inputs + n_inputs));
    struct stat st;
    if (stat(dir.c_str(), &st) == 0 && !S_ISDIR(st.st_mode)) return set_error(nullptr, AC_EINPUT, dir + " exists but is not a directory");
    if (!make_dirs(dir)) return set_error(nullptr, AC_EINPUT, "failed to create directory " + dir + "\n" + strerror(errno));
    if (verbose) {
        fprintf(stderr, "\nStarting autocycler unassembled\n    This command finds the reads the assembly does not explain and the depth of the sequence it "
                        "misses, counted on the GPU. It is not in the reference.\n\nSettings:\n  --reads %s\n  --assemblies", in.c_str());
        for (const std::string& p : paths) fprintf(stderr, " %s", p.c_str());
        fprintf(stderr, "\n  --out_dir %s\n  --kmer %u\n", dir.c_str(), k);
        if (min_count) fprintf(stderr, "  --min_count %u\n", *min_count);
        fprintf(stderr, "  --min_solid %llu\n  --min_fraction %s\n\n", (unsigned long long)min_solid, format_float(min_fraction).c_str());
    }
    UnassembledResult r;
    {
        std::lock_guard<std::mutex> lock(g_subsample_mu);
        SubsampleDevice& d = subsample_device(device);
        try {
            unassembled_run(d.sub, d.spec, d.unassembled, paths, in, k, min_count, min_solid, min_fraction, subsample_window_size(), dir, r);
        } catch (const AcIoError& e) { return set_error(nullptr, AC_EIO, e.msg); }
        catch (const std::length_error& e) { return set_error(nullptr, AC_ERANGE, e.what()); }
    }
    const auto t0 = std::chrono::steady_clock::now();
    const std::pair<std::string, std::string> files[] = {{"unassembled.tsv", r.table}, {"fraction_histogram.tsv", unassembled_fractions(r)},
                                                         {"absent_histogram.tsv", unassembled_absent(r)},
                                                         {"kmer_histogram.tsv", unassembled_kmer_histogram(r)}, {"summary.tsv", unassembled_summary(r)}};
    for (const auto& f : files)
        if (!write_file(dir + "/" + f.first, f.second)) return set_error(nullptr, AC_EIO, "cannot write " + dir + "/" + f.first);
    r.write_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (verbose) {
        fprintf(stderr, "Unassembled reads (k = %u):\n  reads: %llu\n  read k-mer windows: %llu\n  valley: %s\n  min_count: %llu%s\n"
                        "  k-mer depth peak: %s\n  assembly k-mer windows: %llu\n  scored reads: %llu\n  selected reads: %llu (%llu bases)\n"
                        "  absent k-mers: %llu\n  absent k-mer median count: %s\n  absent copy ratio: %s\n\n", k, (unsigned long long)r.reads,
                (unsigned long long)r.read_windows, r.valley ? std::to_string(r.valley).c_str() : "none", (unsigned long long)r.min_count,
                min_count ? " (given)" : " (the valley)", r.has_peak ? unassembled_peak_text(r).c_str() : "none",
                (unsigned long long)r.device.assembly_windows, (unsigned long long)r.scored, (unsigned long long)r.selected,
                (unsigned long long)r.selected_bases, (unsigned long long)r.absent_kmers, r.has_median ? unassembled_median_text(r).c_str() : "none",
                r.has_median && r.has_peak ? unassembled_ratio_text(r).c_str() : "none");
        fprintf(stderr, "Finished!\nUnassembled reads: %s/unassembled.fastq\n\n", dir.c_str());
    }
    if (info) {
        *info = ac_unassembled_info{};
        info->assemblies = r.paths.size(); info->contigs = r.contigs; info->k = k; info->min_count = (uint32_t)r.min_count;
        info->valley = r.valley; info->reads = r.reads; info->read_windows = r.read_windows; info->read_bases = r.read_bases;
        info->distinct = r.distinct; info->scored_reads = r.scored; info->selected_reads = r.selected; info->selected_bases = r.selected_bases;
        info->absent_kmers = r.absent_kmers; info->absent_median = r.has_median ? r.absent_median : NAN; info->peak = r.has_peak ? r.peak : NAN;
        info->absent_copy_ratio = r.has_median && r.has_peak ? r.absent_median / r.peak : NAN;
        info->assembly_windows = r.device.assembly_windows; info->table_bytes = r.device.table_bytes; info->read_bytes = r.device.read_bytes;
        info->spectrum_table_bytes = r.spectrum.table_bytes; info->partitions = r.spectrum.partitions;
        info->reruns = r.spectrum.reruns + r.device.sweep.reruns; info->read_passes = r.selected && r.windows > 1 ? 2 : 1;
        info->kernel_ms = r.kernel_ms; info->scan_ms = r.scan_ms; info->pack_ms = r.pack_reads_ms + r.device.index_ms;
        info->claim_ms = r.device.pack_ms + r.device.claim_ms; info->count_ms = r.spectrum.count_ms + r.spectrum.hist_ms;
        info->sweep_ms = r.device.sweep.count_ms + r.device.attribute_ms; info->gather_ms = r.gather_ms;
        info->read_ms = r.read_ms; info->copy_ms = r.copy_ms; info->write_ms = r.write_ms;
    }
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

// ---- `autocycler polish`: the consensus corrected where the reads' k-mers do not support it (not in the reference) ----------------------
int ac_polish_fasta(const char* reads, const char* assembly, const char* out_dir, uint32_t k, const uint32_t* min_count, uint32_t max_indel,
                    uint32_t rounds, int32_t device, int32_t verbose, ac_polish_info* info) {
    if (!reads || !assembly || !out_dir) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    const std::string in = reads, fasta = assembly, dir = out_dir;
    if (k < 11 || k > 31 || k % 2 == 0) return set_error(nullptr, AC_EINPUT, "--kmer must be odd and between 11 and 31");
    if (min_count && (*min_count < 1 || *min_count > AC_GS_BINS - 1))
        return set_error(nullptr, AC_EINPUT, "--min_count must be between 1 and " + std::to_string(AC_GS_BINS - 1));
    if (max_indel < 1 || max_indel > 4) return set_error(nullptr, AC_EINPUT, "--max_indel must be between 1 and 4");
    if (rounds < 1 || rounds > 10) return set_error(nullptr, AC_EINPUT, "--rounds must be between 1 and 10");
    int rc;
    if ((rc = check_file(in)) != AC_OK) return rc;
    if ((rc = check_file(fasta)) != AC_OK) return rc;
    struct stat st;
    if (stat(dir.c_str(), &st) == 0 && !S_ISDIR(st.st_mode)) return set_error(nullptr, AC_EINPUT, dir + " exists but is not a directory");
    if (!make_dirs(dir)) return set_error(nullptr, AC_EINPUT, "failed to create directory " + dir + "\n" + strerror(errno));
    if (verbose) {
        fprintf(stderr, "\nStarting autocycler polish\n    This command corrects the consensus where the reads' k-mers do not support it, with "
                        "candidate edits scored on the GPU. It is not in the reference.\n\nSettings:\n  --reads %s\n  --input %s\n  --out_dir %s\n"
                        "  --kmer %u\n", in.c_str(), fasta.c_str(), dir.c_str(), k);
        if (min_count) fprintf(stderr, "  --min_count %u\n", *min_count);
        fprintf(stderr, "  --max_indel %u\n  --rounds %u\n\n", max_indel, rounds);
    }
    PolishResult r;
    {
        std::lock_guard<std::mutex> lock(g_subsample_mu);
        SubsampleDevice& d = subsample_device(device);
        try {
            polish_run(d.sub, d.spec, d.polish, fasta, in, k, min_count, max_indel, rounds, subsample_window_size(), r);
        } catch (const AcIoError& e) { return set_error(nullptr, AC_EIO, e.msg); }
        catch (const std::length_error& e) { return set_error(nullptr, AC_ERANGE, e.what()); }
    }
    const auto t0 = std::chrono::steady_clock::now();
    const std::pair<std::string, std::string> files[] = {{"polished.fasta", polish_fasta(r)}, {"edits.tsv", polish_edits(r)},
                                                         {"rounds.tsv", polish_rounds(r)}, {"remaining.bed", r.bed},
                                                         {"summary.tsv", polish_summary(r, k)}};
    for (const auto& f : files)
        if (!write_file(dir + "/" + f.first, f.second)) return set_error(nullptr, AC_EIO, "cannot write " + dir + "/" + f.first);
    const double write_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (verbose) {
        fprintf(stderr, "K-mer polish (k = %u):\n  reads: %llu\n  read k-mer windows: %llu\n  valley: %s\n  min_count: %llu%s\n", k,
                (unsigned long long)r.reads, (unsigned long long)r.read_windows, r.valley ? std::to_string(r.valley).c_str() : "none",
                (unsigned long long)r.min_count, min_count ? " (given)" : " (the valley)");
        for (size_t i = 0; i < r.rounds.size(); ++i) {
            const PolishRound& x = r.rounds[i];
            fprintf(stderr, "  round %zu: %llu unsupported k-mers, %llu loci: %llu edited, %llu ambiguous, %llu none, %llu edge, %llu deferred\n",
                    i + 1, (unsigned long long)x.unsupported, (unsigned long long)x.loci, (unsigned long long)x.edited,
                    (unsigned long long)x.ambiguous, (unsigned long long)x.none, (unsigned long long)x.edge, (unsigned long long)x.deferred);
        }
        fprintf(stderr, "  QV: %s before, %s after (%llu edits)\n\nFinished!\nPolished assembly: %s/polished.fasta\n\n",
                qv_text(r.unsupported_before, r.kmers_before, k).c_str(), qv_text(r.unsupported_after, r.kmers_after, k).c_str(),
                (unsigned long long)r.edits, dir.c_str());
    }
    if (info) {
        *info = ac_polish_info{};
        info->contigs = r.recs.size(); info->k = k; info->min_count = (uint32_t)r.min_count; info->valley = r.valley;
        info->reads = r.reads; info->read_windows = r.read_windows; info->read_bases = r.read_bases; info->distinct = r.distinct;
        info->kmers_before = r.kmers_before; info->unsupported_before = r.unsupported_before; info->kmers_after = r.kmers_after;
        info->unsupported_after = r.unsupported_after; info->edits = r.edits; info->rounds = r.rounds.size();
        for (const PolishRound& x : r.rounds) info->loci += x.loci;
        info->table_bytes = r.device.table_bytes; info->candidate_table_bytes = r.device.candidate_bytes; info->batches = r.device.batches;
        info->spectrum_table_bytes = r.spectrum.table_bytes; info->partitions = r.spectrum.partitions;
        info->reruns = r.spectrum.reruns + r.device.sweep.reruns;
        info->kernel_ms = r.kernel_ms; info->scan_ms = r.scan_ms; info->pack_ms = r.pack_reads_ms; info->count_ms = r.spectrum.count_ms + r.spectrum.hist_ms;
        info->contig_ms = r.device.pack_ms; info->fill_ms = r.device.fill_ms; info->recount_ms = r.device.sweep.count_ms;
        info->candidate_ms = r.device.candidate_ms; info->choose_ms = r.device.choose_ms;
        info->read_ms = r.read_ms; info->copy_ms = r.copy_ms; info->host_ms = r.host_ms; info->write_ms = write_ms;
    }
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

// ---- `autocycler variants`: the alleles the reads carry beside the consensus (not in the reference) -------------------------------------
int ac_variants_fasta(const char* reads, const char* assembly, const char* out_dir, uint32_t k, const uint32_t* min_count, uint32_t max_indel,
                      double min_fraction, int32_t device, int32_t verbose, ac_variants_info* info) {
    if (!reads || !assembly || !out_dir) return set_error(nullptr, AC_EINVAL, "null argument");
    AC_GUARD_BEGIN
    const std::string in = reads, fasta = assembly, dir = out_dir;
    if (k < 11 || k > 31 || k % 2 == 0) return set_error(nullptr, AC_EINPUT, "--kmer must be odd and between 11 and 31");
    if (min_count && (*min_count < 1 || *min_count > AC_GS_BINS - 1))
        return set_error(nullptr, AC_EINPUT, "--min_count must be between 1 and " + std::to_string(AC_GS_BINS - 1));
    if (max_indel > 3) return set_error(nullptr, AC_EINPUT, "--max_indel must be between 0 and 3");
    if (!(min_fraction > 0.0 && min_fraction <= 1.0)) return set_error(nullptr, AC_EINPUT, "--min_fraction must be above 0 and at most 1");
    int rc;
    if ((rc = check_file(in)) != AC_OK) return rc;
    if ((rc = check_file(fasta)) != AC_OK) return rc;
    struct stat st;
    if (stat(dir.c_str(), &st) == 0 && !S_ISDIR(st.st_mode)) return set_error(nullptr, AC_EINPUT, dir + " exists but is not a directory");
    if (!make_dirs(dir)) return set_error(nullptr, AC_EINPUT, "failed to create directory " + dir + "\n" + strerror(errno));
    if (verbose) {
        fprintf(stderr, "\nStarting autocycler variants\n    This command finds the alleles the reads carry beside the consensus, with every "
                        "position's alternatives screened on the GPU. It is not in the reference.\n\nSettings:\n  --reads %s\n  --input %s\n"
                        "  --out_dir %s\n  --kmer %u\n", in.c_str(), fasta.c_str(), dir.c_str(), k);
        if (min_count) fprintf(stderr, "  --min_count %u\n", *min_count);
        fprintf(stderr, "  --max_indel %u\n  --min_fraction %s\n\n", max_indel, format_float(min_fraction).c_str());
    }
    VariantsResult r;
    {
        std::lock_guard<std::mutex> lock(g_subsample_mu);
        SubsampleDevice& d = subsample_device(device);
        try {
            variants_run(d.sub, d.spec, d.polish, d.variants, fasta, in, k, min_count, max_indel, min_fraction, subsample_window_size(), r);
        } catch (const AcIoError& e) { return set_error(nullptr, AC_EIO, e.msg); }
        catch (const std::length_error& e) { return set_error(nullptr, AC_ERANGE, e.what()); }
    }
    const auto t0 = std::chrono::steady_clock::now();
    const std::pair<std::string, std::string> files[] = {{"variants.vcf", variants_vcf(r)}, {"summary.tsv", variants_summary(r)}};
    for (const auto& f : files)
        if (!write_file(dir + "/" + f.first, f.second)) return set_error(nullptr, AC_EIO, "cannot write " + dir + "/" + f.first);
    const double write_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (verbose) {
        fprintf(stderr, "K-mer variants (k = %u):\n  reads: %llu\n  read k-mer windows: %llu\n  valley: %s\n  min_count: %llu%s\n"
                        "  positions: %llu\n  screened: %llu\n  candidates: %llu (%llu passing)\n  variants: %llu (%llu substitutions, %llu insertions, "
                        "%llu deletions)\n  paralog: %llu\n  alt_major: %llu\n\nFinished!\nVariants: %s/variants.vcf\n\n", k,
                (unsigned long long)r.reads, (unsigned long long)r.read_windows, r.valley ? std::to_string(r.valley).c_str() : "none",
                (unsigned long long)r.min_count, min_count ? " (given)" : " (the valley)", (unsigned long long)r.positions,
                (unsigned long long)r.screened, (unsigned long long)r.candidates, (unsigned long long)r.passing, (unsigned long long)r.rows.size(),
                (unsigned long long)r.substitutions, (unsigned long long)r.insertions, (unsigned long long)r.deletions,
                (unsigned long long)r.paralog, (unsigned long long)r.alt_major, dir.c_str());
    }
    if (info) {
        *info = ac_variants_info{};
        info->contigs = r.recs.size(); info->k = k; info->min_count = (uint32_t)r.min_count; info->valley = r.valley;
        info->reads = r.reads; info->read_windows = r.read_windows; info->read_bases = r.read_bases; info->distinct = r.distinct;
        info->kmers = r.kmers; info->positions = r.positions; info->screened = r.screened; info->candidates = r.candidates;
        info->loci = r.loci; info->passing = r.passing; info->variants = r.rows.size(); info->substitutions = r.substitutions;
        info->insertions = r.insertions; info->deletions = r.deletions; info->paralog = r.paralog; info->alt_major = r.alt_major;
        info->table_bytes = r.device.table_bytes; info->candidate_table_bytes = r.device.candidate_bytes; info->batches = r.device.batches;
        info->spectrum_table_bytes = r.spectrum.table_bytes; info->partitions = r.spectrum.partitions;
        info->reruns = r.spectrum.reruns + r.device.sweep.reruns;
        info->kernel_ms = r.kernel_ms; info->scan_ms = r.scan_ms; info->pack_ms = r.pack_reads_ms; info->count_ms = r.spectrum.count_ms + r.spectrum.hist_ms;
        info->contig_ms = r.device.pack_ms; info->fill_ms = r.device.fill_ms; info->screen_ms = r.va.screen_ms; info->recount_ms = r.device.sweep.count_ms;
        info->candidate_ms = r.device.candidate_ms; info->ref_ms = r.va.ref_ms;
        info->read_ms = r.read_ms; info->copy_ms = r.copy_ms; info->host_ms = r.host_ms; info->write_ms = write_ms;
    }
    return ok(nullptr);
    AC_GUARD_END(nullptr)
}

}  // extern "C"
