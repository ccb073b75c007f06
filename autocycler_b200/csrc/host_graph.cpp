// Host side of the compress path (see host_graph.h).  Citations are file:line in the reference's src/.
#include "host_graph.h"

#include <algorithm>
#include <atomic>
#include <charconv>
#include <chrono>
#include <cstring>
#include <condition_variable>
#include <mutex>
#include <stdexcept>
#include <thread>
#include <type_traits>
#include <unistd.h>

namespace {
inline double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

inline char comp(char c) {   // misc.rs:324-333 (unitig sequences hold only ACGT after trimming)
    switch (c) { case 'A': return 'T'; case 'T': return 'A'; case 'C': return 'G'; case 'G': return 'C'; default: return c == '.' ? '.' : 'N'; }
}

unsigned host_threads() {
    static const unsigned n = [] {
        unsigned hw = std::thread::hardware_concurrency();
        if (const char* e = getenv("AC_HOST_THREADS")) { int v = atoi(e); if (v > 0) return (unsigned)v; }
        return hw == 0 ? 4u : (hw > 48 ? 48u : hw);   // at most 48: the host stages of the largest configs stop gaining well before that
    }();
    return n;
}

// Persistent worker threads for parallel_tasks: the host stages issue a few dozen short parallel regions per graph, and
// spawning + joining 15 threads for each of them costs more than several of the regions themselves.  Workers spin briefly
// after a job (the next region usually follows within microseconds) and then sleep on a condition variable.
class WorkerPool {
public:
    static WorkerPool& get() { static WorkerPool pool; return pool; }
    // Runs job(ctx) on the caller and on `helpers` workers; returns when all of them have left the job.
    void run(unsigned helpers, void (*job)(void*), void* ctx) {
        std::lock_guard<std::mutex> one_job_at_a_time(entry);
        {
            std::lock_guard<std::mutex> lk(m);
            if (owner != getpid()) { new std::vector<std::thread>(std::move(workers)); workers.clear(); owner = getpid(); }   // after fork(): the threads stayed behind
            while (workers.size() < helpers) { const unsigned id = (unsigned)workers.size(); workers.emplace_back([this, id] { loop(id); }); }
            fn = job; arg = ctx; wanted = helpers;
            pending.store(helpers, std::memory_order_relaxed);
            generation.fetch_add(1, std::memory_order_release);
        }
        cv.notify_all();
        job(ctx);
        for (unsigned spins = 0; pending.load(std::memory_order_acquire) != 0; ++spins) { if (spins > 2000) std::this_thread::yield(); }
    }
    ~WorkerPool() {
        { std::lock_guard<std::mutex> lk(m); stopping = true; generation.fetch_add(1, std::memory_order_release); }
        cv.notify_all();
        if (owner == getpid()) for (auto& w : workers) w.join();
        else new std::vector<std::thread>(std::move(workers));
    }
private:
    void loop(unsigned id) {
        uint64_t seen = 0;
        for (;;) {
            const auto spin_until = std::chrono::steady_clock::now() + std::chrono::microseconds(200);
            while (generation.load(std::memory_order_acquire) == seen && std::chrono::steady_clock::now() < spin_until) {}
            void (*job)(void*); void* ctx; bool mine;
            {
                std::unique_lock<std::mutex> lk(m);
                cv.wait(lk, [&] { return generation.load(std::memory_order_relaxed) != seen; });
                if (stopping) return;
                seen = generation.load(std::memory_order_relaxed);
                job = fn; ctx = arg; mine = id < wanted;
            }
            if (!mine) continue;
            job(ctx);
            pending.fetch_sub(1, std::memory_order_release);
        }
    }
    std::mutex entry, m;
    std::condition_variable cv;
    std::vector<std::thread> workers;
    std::atomic<uint64_t> generation{0};
    std::atomic<unsigned> pending{0};
    void (*fn)(void*) = nullptr; void* arg = nullptr; unsigned wanted = 0; bool stopping = false;
    pid_t owner = getpid();
};

// Runs fn() exactly once on each of T threads (the caller and T-1 workers): for loops with their own barriers.
template <class F> void run_on_threads(unsigned T, F& fn) {
    if (T <= 1) { fn(); return; }
    WorkerPool::get().run(T - 1, [](void* p) { (*static_cast<F*>(p))(); }, &fn);
}

// Runs fn(task) for task in [0, n_tasks) on up to host_threads() threads (dynamic scheduling).
template <class F> void parallel_tasks(size_t n_tasks, F&& fn) {
    static thread_local bool inside = false;
    const unsigned nt = inside ? 1u : (unsigned)std::min<size_t>(host_threads(), n_tasks);
    if (nt <= 1) { for (size_t t = 0; t < n_tasks; ++t) fn(t); return; }
    struct Job {
        std::remove_reference_t<F>* fn; size_t n_tasks; std::atomic<size_t> next{0};
        std::exception_ptr err = nullptr; std::atomic<bool> failed{false};
    } job;
    job.fn = &fn; job.n_tasks = n_tasks;
    auto work = [](void* p) {
        Job& j = *static_cast<Job*>(p);
        inside = true;
        try { for (size_t t; (t = j.next.fetch_add(1)) < j.n_tasks;) (*j.fn)(t); }
        catch (...) { if (!j.failed.exchange(true)) j.err = std::current_exception(); }
        inside = false;
    };
    static const bool pooled = !(getenv("AC_HOST_POOL") && atoi(getenv("AC_HOST_POOL")) == 0);
    if (pooled) WorkerPool::get().run(nt - 1, work, &job);
    else {                                   // one-shot threads (kept for comparison)
        std::vector<std::thread> once;
        for (unsigned t = 1; t < nt; ++t) once.emplace_back(work, &job);
        work(&job);
        for (auto& th : once) th.join();
    }
    if (job.err) std::rethrow_exception(job.err);
}
}  // namespace

// ------------------------------------------------------------------------------------------------
// build: adopt the device result (already in seed order, links already in the reference's push order)
// ------------------------------------------------------------------------------------------------
void HostGraph::build(const PipelineResult& r, const std::vector<HostSeq>& seqs, uint32_t k_size, bool keep_positions) {
    prof = HostProfile();
    const double t0 = now_ms();
    k = k_size;
    U = r.n_unitigs;
    fixed_ready = false; cands_ready = false;
    rec = r.rec; depth = r.depth; depth_f = nullptr; utype = nullptr;
    arena = r.arena; arena_used = r.arena_used; arena_cap = r.arena_cap; arena_overflow.clear();
    next_off = r.next_off; next = r.next; prev_off = r.prev_off; prev = r.prev; n_links = r.n_links;
    path_off = r.path_off; path = r.path; n_path = r.n_runs; n_seqs = r.n_seqs;
    number.assign(U, 0);

    // Full position lists (unitig.rs:135-146), only on request: an occurrence [fs, fs+n) on the forward strand of
    // sequence i is also an occurrence of the opposite unitig strand at L-fs-n on its reverse strand (kmer_graph.rs:103-108).
    fpos_off.clear(); rpos_off.clear(); fpos.clear(); rpos.clear();
    if (keep_positions) {
        const size_t R = r.n_runs, S = seqs.size();
        std::vector<uint32_t> pos_count(U, 0);
        for (size_t x = 0; x < R; ++x) pos_count[us_index(path[x])] += 1;
        fpos_off.assign((size_t)U + 1, 0);
        for (uint32_t u = 0; u < U; ++u) fpos_off[u + 1] = fpos_off[u] + pos_count[u];
        rpos_off = fpos_off; fpos.resize(R); rpos.resize(R);
        std::vector<uint64_t> cursor(fpos_off.begin(), fpos_off.end() - 1);
        size_t si = 0;
        for (size_t x = 0; x < R; ++x) {
            const uint64_t g = r.run_start[x];
            while (si + 1 < S && seqs[si + 1].start <= g) ++si;
            const HostSeq& s = seqs[si];
            const UStrand p = path[x]; const bool plus = !us_reverse(p); const uint32_t idx = us_index(p);
            const uint32_t fs = (uint32_t)(g - s.start), n = r.run_len[x], mirrored = (uint32_t)(s.length - fs - n);
            const uint64_t at = cursor[idx]++;
            fpos[at] = ((uint64_t)(plus ? fs : mirrored) << 16) | (uint64_t)(s.id | (plus ? 0x8000u : 0u));
            rpos[at] = ((uint64_t)(plus ? mirrored : fs) << 16) | (uint64_t)(s.id | (plus ? 0u : 0x8000u));
        }
    }
    prof.adopt = now_ms() - t0;

    order.resize(U);
    // sorted on the device while the sequences were still in HBM: the numbering of the graph as built or, after a fused build, the one
    // simplify_structure ends with (graph_simplification.rs:38)
    const uint32_t* given = r.final_order ? r.final_order : r.order;
    if (given) {
        const double t1 = now_ms();
        memcpy(order.data(), given, (size_t)U * 4);
        for (uint32_t n = 0; n < U; ++n) number[order[n]] = n + 1;
        prof.renumber += now_ms() - t1;
    } else {
        for (uint32_t s = 0; s < U; ++s) order[s] = s;
        renumber();
    }
}

// ------------------------------------------------------------------------------------------------
// renumber / checks / counts
// ------------------------------------------------------------------------------------------------
void HostGraph::renumber() {   // unitig_graph.rs:295-315: stable sort by length desc, sequence asc, depth desc
    const double t0 = now_ms();
    struct Key { uint32_t len; uint32_t pos; uint64_t prefix; uint32_t idx; double depth; };
    std::vector<Key> keys(U);
    const size_t T = std::max<size_t>(1, std::min<size_t>(host_threads(), U / 4096));
    auto bounds = [&](size_t t) { return (size_t)((uint64_t)U * t / T); };
    auto less = [&](const Key& a, const Key& b) {
        if (a.len != b.len) return a.len > b.len;
        if (a.prefix != b.prefix) return a.prefix < b.prefix;
        if (a.len > 8) { const int c = memcmp(seq_ptr(a.idx) + 8, seq_ptr(b.idx) + 8, a.len - 8); if (c != 0) return c < 0; }
        if (a.depth != b.depth) return a.depth > b.depth;
        return a.pos < b.pos;   // ties keep their previous order: slice::sort_by is stable
    };
    parallel_tasks(T, [&](size_t t) {
        for (size_t n = bounds(t); n < bounds(t + 1); ++n) {
            const uint32_t idx = order[n];
            Key& key = keys[n];
            key.len = rec[idx].len; key.pos = (uint32_t)n; key.idx = idx; key.depth = depth_of(idx);
            const unsigned char* p = (const unsigned char*)seq_ptr(idx);
            uint64_t v = 0;
            const uint32_t m = key.len < 8 ? key.len : 8;
            for (uint32_t i = 0; i < m; ++i) v |= (uint64_t)p[i] << (56 - 8 * i);
            key.prefix = v;
        }
    });
    const double t_keys = now_ms();
    if (T == 1) std::sort(keys.begin(), keys.end(), less);
    else {   // sample sort: splitters from a sample, every thread scatters its piece into the buckets, every bucket is sorted on its own
        const size_t B = T, per = 16;
        std::vector<Key> sample;
        for (size_t x = 0; x < B * per; ++x) sample.push_back(keys[(size_t)((uint64_t)U * x / (B * per))]);
        std::sort(sample.begin(), sample.end(), less);
        std::vector<Key> split;
        for (size_t b = 1; b < B; ++b) split.push_back(sample[b * per]);
        auto bucket_of = [&](const Key& key) { return (size_t)(std::upper_bound(split.begin(), split.end(), key, less) - split.begin()); };
        std::vector<uint32_t> count(T * B, 0);
        std::vector<uint8_t> which(U);
        parallel_tasks(T, [&](size_t t) {
            for (size_t n = bounds(t); n < bounds(t + 1); ++n) { const size_t b = bucket_of(keys[n]); which[n] = (uint8_t)b; count[t * B + b] += 1; }
        });
        std::vector<uint32_t> at(T * B), bucket_start(B + 1, 0);
        { uint32_t run = 0; for (size_t b = 0; b < B; ++b) { bucket_start[b] = run; for (size_t t = 0; t < T; ++t) { at[t * B + b] = run; run += count[t * B + b]; } } bucket_start[B] = run; }
        std::vector<Key> sorted(U);
        parallel_tasks(T, [&](size_t t) {
            for (size_t n = bounds(t); n < bounds(t + 1); ++n) sorted[at[t * B + which[n]]++] = keys[n];
        });
        parallel_tasks(B, [&](size_t b) { std::sort(sorted.begin() + bucket_start[b], sorted.begin() + bucket_start[b + 1], less); });
        keys.swap(sorted);
    }
    const double t_sort = now_ms();
    parallel_tasks(T, [&](size_t t) { for (size_t n = bounds(t); n < bounds(t + 1); ++n) { order[n] = keys[n].idx; number[keys[n].idx] = (uint32_t)n + 1; } });
    prof.renumber += now_ms() - t0;
    if (getenv("AC_HOST_PROFILE")) fprintf(stderr, "[host] renumber: keys %.2f, sort %.2f, write %.2f ms (%zu threads)\n", t_keys - t0, t_sort - t_keys, now_ms() - t_sort, T);
}

void HostGraph::check_links() const {   // unitig_graph.rs:752-793: every link has its mirror and its prev entry
    auto has = [](const UStrand* b, uint32_t n, UStrand x) { for (uint32_t i = 0; i < n; ++i) if (b[i] == x) return true; return false; };
    const size_t n_strands = 2 * (size_t)U, T = std::max<size_t>(1, std::min<size_t>(host_threads(), n_strands / 8192));
    parallel_tasks(T, [&](size_t t) {
        for (UStrand from = (UStrand)(n_strands * t / T); from < (UStrand)(n_strands * (t + 1) / T); ++from) {
            for (uint32_t x = next_off[from]; x < next_off[from + 1]; ++x) {
                const UStrand to = next[x];
                if (!has(prev_begin(to), prev_size(to), from)) throw std::runtime_error("missing prev link");
                if (!has(next_begin(us_flip(to)), next_size(us_flip(to)), us_flip(from))) throw std::runtime_error("missing next link");
            }
            for (uint32_t x = prev_off[from]; x < prev_off[from + 1]; ++x)
                if (!has(next_begin(prev[x]), next_size(prev[x]), from)) throw std::runtime_error("missing next link");
        }
    });
}

uint64_t HostGraph::total_length() const { uint64_t t = 0; for (uint32_t u = 0; u < U; ++u) t += rec[u].len; return t; }

uint64_t HostGraph::link_count_single() const {   // unitig_graph.rs:478-507: a link and its mirror count once; hairpins are their own mirror
    uint64_t all = n_links, hairpins = 0;
    for (UStrand from = 0; from < 2 * U; ++from)
        for (uint32_t x = next_off[from]; x < next_off[from + 1]; ++x) if (next[x] == us_flip(from)) ++hairpins;
    return (all - hairpins) / 2 + hairpins;
}

// ------------------------------------------------------------------------------------------------
// arena growth
// ------------------------------------------------------------------------------------------------
void HostGraph::reserve_arena(uint64_t extra) {   // make room for `extra` more bytes (single-threaded)
    if (arena_used + extra <= arena_cap) return;
    std::vector<char> bigger((arena_used + extra) * 2);
    memcpy(bigger.data(), arena, arena_used);
    arena_overflow.swap(bigger);
    arena = arena_overflow.data(); arena_cap = arena_overflow.size();
}
bool HostGraph::relocate(uint32_t idx, uint32_t before, uint32_t after, bool shared) {
    const uint64_t need = (uint64_t)before + rec[idx].len + after;
    uint64_t at = __atomic_fetch_add(&arena_used, need, __ATOMIC_RELAXED);
    if (at + need > arena_cap) {
        __atomic_fetch_sub(&arena_used, need, __ATOMIC_RELAXED);
        if (shared) return false;             // other threads hold pointers into the arena: it cannot move now
        reserve_arena(need);
        at = arena_used; arena_used += need;
    }
    memmove(arena + at + before, arena + rec[idx].seq_off, rec[idx].len);
    rec[idx].seq_off = at + before; rec[idx].room_before = before; rec[idx].room_after = after;
    return true;
}

// ------------------------------------------------------------------------------------------------
// graph_simplification.rs:26-312
// ------------------------------------------------------------------------------------------------
void HostGraph::compute_fixed() {   // graph_simplification.rs:190-230; paths and links never change during simplification
    fixed_start.assign(U, 0); fixed_end.assign(U, 0);
    for (size_t i = 0; i < n_seqs; ++i) {
        if (path_off[i + 1] == path_off[i]) continue;
        const UStrand first = path[path_off[i]], last = path[path_off[i + 1] - 1];
        if (!us_reverse(first)) fixed_start[us_index(first)] = 1; else fixed_end[us_index(first)] = 1;
        if (!us_reverse(last)) fixed_end[us_index(last)] = 1; else fixed_start[us_index(last)] = 1;
    }
    const std::vector<uint8_t> starts_copy = fixed_start, ends_copy = fixed_end;
    for (uint32_t u = 0; u < U; ++u) {
        if (starts_copy[u]) {
            const UStrand s = us_make(u, false);
            for (uint32_t x = prev_off[s]; x < prev_off[s + 1]; ++x) { const UStrand up = prev[x]; if (!us_reverse(up)) fixed_end[us_index(up)] = 1; else fixed_start[us_index(up)] = 1; }
        }
        if (ends_copy[u]) {
            const UStrand s = us_make(u, false);
            for (uint32_t x = next_off[s]; x < next_off[s + 1]; ++x) { const UStrand down = next[x]; if (!us_reverse(down)) fixed_start[us_index(down)] = 1; else fixed_end[us_index(down)] = 1; }
        }
    }
    fixed_ready = true;
}

// Which (unitig, side) pairs can ever shift is decided by links, paths and fixed sets alone, and none of those change
// while `while expand_repeats() > 0 {}` runs (graph_simplification.rs:26-27; the renumbering comes after), so the
// candidates are listed once, in the iteration order of the reference's loop (graph.unitigs order; inputs side first).
void HostGraph::compute_candidates() {
    const bool prof_on = getenv("AC_HOST_PROFILE") != nullptr; double tt = now_ms();
    auto lap = [&](const char* what) { if (prof_on) { const double t = now_ms(); fprintf(stderr, "[host]   candidates/%s %.2f ms\n", what, t - tt); tt = t; } };
    if (!fixed_ready) compute_fixed();
    lap("fixed");
    const size_t T = std::max<size_t>(1, std::min<size_t>(host_threads(), U / 8192));
    std::vector<std::vector<Candidate>> part(T);
    parallel_tasks(T, [&](size_t t) {
        std::vector<Candidate>& out = part[t];
        for (uint32_t n = (uint32_t)((uint64_t)U * t / T); n < (uint32_t)((uint64_t)U * (t + 1) / T); ++n) {
            const uint32_t idx = order[n];
            const UStrand self_fwd = us_make(idx, false);
            {   // get_exclusive_inputs (:233-255) and the guards of expand_repeats (:66-72)
                const UStrand* grp = prev_begin(self_fwd); const uint32_t gn = prev_size(self_fwd);
                bool ok = gn >= 2 && !fixed_start[idx];
                for (uint32_t a = 0; ok && a < gn; ++a) {
                    const UStrand p = grp[a];
                    if (!(next_size(p) == 1 && next_begin(p)[0] == self_fwd) || us_index(p) == idx) ok = false;
                    else if ((!us_reverse(p) && fixed_end[us_index(p)]) || (us_reverse(p) && fixed_start[us_index(p)])) ok = false;
                }
                if (ok) { Candidate c{idx, 0, (uint16_t)gn, {0, 0, 0, 0, 0, 0}}; for (uint32_t a = 0; a < gn && a < 6; ++a) c.src[a] = grp[a]; out.push_back(c); }
            }
            {   // get_exclusive_outputs (:258-280) and the guards (:75-82)
                const UStrand* grp = next_begin(self_fwd); const uint32_t gn = next_size(self_fwd);
                bool ok = gn >= 2 && !fixed_end[idx];
                for (uint32_t a = 0; ok && a < gn; ++a) {
                    const UStrand q = grp[a];
                    if (!(prev_size(q) == 1 && prev_begin(q)[0] == self_fwd) || us_index(q) == idx) ok = false;
                    else if ((!us_reverse(q) && fixed_start[us_index(q)]) || (us_reverse(q) && fixed_end[us_index(q)])) ok = false;
                }
                if (ok) { Candidate c{idx, 1, (uint16_t)gn, {0, 0, 0, 0, 0, 0}}; for (uint32_t a = 0; a < gn && a < 6; ++a) c.src[a] = grp[a]; out.push_back(c); }
            }
        }
    });
    lap("list");
    std::vector<size_t> part_at(T + 1, 0);
    for (size_t t = 0; t < T; ++t) part_at[t + 1] = part_at[t] + part[t].size();
    cands.resize(part_at[T]);
    cand_at.resize(2 * (size_t)U);
    parallel_tasks(T, [&](size_t t) {                    // the pieces are in graph order already: copy them side by side and index them
        const size_t a = (size_t)((uint64_t)U * t / T), b = (size_t)((uint64_t)U * (t + 1) / T);
        for (size_t n = a; n < b; ++n) { cand_at[2 * (size_t)order[n]] = -1; cand_at[2 * (size_t)order[n] + 1] = -1; }
        for (size_t x = 0; x < part[t].size(); ++x) {
            const Candidate& c = part[t][x];
            cands[part_at[t] + x] = c;
            cand_at[2 * (size_t)c.idx + c.side] = (int32_t)(part_at[t] + x);
        }
    });
    lap("concat+index");
    compute_dependents();
    lap("dependents");
    compute_levels();
    lap("levels");
    dirty.assign((cands.size() + 63) / 64, 0);     // the first pass visits every candidate; the bitmap collects work for later passes
    exhausted.assign(cands.size(), 0);
    for (uint32_t u = 0; u < U; ++u) rec[u].flags = 0;
    first_pass = true;
    cands_ready = true; spec_from_device = false;
}

namespace {
const struct CompLut { unsigned char same[256], comp[256]; CompLut() { for (int i = 0; i < 256; ++i) { same[i] = (unsigned char)i; comp[i] = (unsigned char)::comp((char)i); } } } g_lut;
// A unitig strand read from its start or from its end without materialising the reverse complement
// (UnitigStrand::get_seq): character i is map[base[i * step]].
struct Cursor { const unsigned char* base; ptrdiff_t step; const unsigned char* map;
                unsigned char at(size_t i) const { return map[base[(ptrdiff_t)i * step]]; } };
}  // namespace

// get_common_end_seq (:298-312) for side 0 / get_common_start_seq (:283-295) for side 1: length of the common piece
uint32_t HostGraph::common_length(const Candidate& cand) const {
    const UStrand* grp = sources(cand); const uint32_t gn = cand.gn;
    auto cursor = [&](UStrand s) {
        const uint32_t u = us_index(s); const unsigned char* p = (const unsigned char*)seq_ptr(u);
        const bool at_back = (cand.side == 0) != us_reverse(s);    // forward strand read from its end, or reverse strand read from its start
        return Cursor{at_back ? p + rec[u].len - 1 : p, at_back ? -1 : 1, us_reverse(s) ? g_lut.comp : g_lut.same};
    };
    const Cursor first = cursor(grp[0]);
    size_t c = rec[us_index(grp[0])].len;
    for (uint32_t a = 1; a < gn; ++a) {
        const uint32_t la = rec[us_index(grp[a])].len;
        if (la < c) c = la;
        const Cursor cur = cursor(grp[a]);
        size_t m = 0;
        while (m < c && cur.at(m) == first.at(m)) ++m;
        c = m;
    }
    return (uint32_t)c;
}

// A change to unitig u can only matter to the candidates that read it: those of u itself (its minimum position) and
// those of the unitigs it exclusively feeds (as an input) or is exclusively fed by (as an output).
void HostGraph::compute_dependents() {
    deps.resize(U);
    const size_t T = std::max<size_t>(1, std::min<size_t>(host_threads(), U / 8192));
    parallel_tasks(T, [&](size_t t) {
        for (uint32_t u = (uint32_t)((uint64_t)U * t / T); u < (uint32_t)((uint64_t)U * (t + 1) / T); ++u) {
            Deps& d = deps[u];
            d.c[0] = cand_at[2 * (size_t)u]; d.c[1] = cand_at[2 * (size_t)u + 1];
            for (uint32_t rev = 0; rev < 2; ++rev) {
                const UStrand s = us_make(u, rev != 0);
                d.c[2 + 2 * rev] = (next_size(s) == 1 && !us_reverse(next_begin(s)[0])) ? cand_at[2 * (size_t)us_index(next_begin(s)[0])] : -1;
                d.c[3 + 2 * rev] = (prev_size(s) == 1 && !us_reverse(prev_begin(s)[0])) ? cand_at[2 * (size_t)us_index(prev_begin(s)[0]) + 1] : -1;
            }
        }
    });
}


// One evaluation of candidate ci: graph_simplification.rs:64-84 for one (unitig, side).  Returns the bases moved.
// `shared` = other threads are applying candidates with disjoint unitig sets at the same time (bitmap and arena bump
// go through atomics).
size_t HostGraph::apply_candidate(size_t ci, bool shared, std::string& common) {
    const size_t w = ci >> 6; const uint64_t bit_mask = 1ull << (ci & 63);
    const Candidate cand = cands[ci];
    const uint32_t idx = cand.idx;
    const UStrand* grp = sources(cand); const uint32_t gn = cand.gn;

    // the comparison made in parallel at the start of this pass still holds if none of the sources changed since
    bool dup = false, pristine = spec_pass[ci] == pass_id; uint32_t min_len = 0xFFFFFFFFu;
    for (uint32_t a = 0; a < gn; ++a) {
        const uint32_t s = us_index(grp[a]);
        if (rec[s].len < min_len) min_len = rec[s].len;
        if (rec[s].flags == pass_id) pristine = false;
        for (uint32_t b = 0; b < a; ++b) if (s == us_index(grp[b])) dup = true;
    }
    const size_t common_len = pristine ? spec_len[ci] : common_length(cand);
    size_t c = common_len;
    // avoid_zero_len_unitigs (:141-158) and avoid_start_of_path (:161-181) trim the common piece on the far side
    if (c > 0) c = std::min<size_t>(c, (min_len - 1) / (dup ? 2 : 1));
    const uint32_t min_pos = cand.side == 0 ? rec[idx].min_fpos : rec[idx].min_rpos;
    if (c > 0) c = min_pos == 0 ? 0 : std::min<size_t>(c, min_pos - 1);
    exhausted[ci] = c == common_len;       // nothing (more) in common: only an extension of a compared end can change that
    if (c == 0) return 0;

    // make room at the destination BEFORE anything is modified: when several threads share the arena it cannot be
    // reallocated, and a candidate that does not fit is handed back untouched (the caller applies it alone later)
    if (cand.side == 0 ? rec[idx].room_before < c : rec[idx].room_after < c) {
        const uint32_t before = cand.side == 0 ? (uint32_t)c + 4 * AC_SEQ_SLACK : std::max<uint32_t>(rec[idx].room_before, AC_SEQ_SLACK);
        const uint32_t after = cand.side == 0 ? std::max<uint32_t>(rec[idx].room_after, AC_SEQ_SLACK) : (uint32_t)c + 4 * AC_SEQ_SLACK;
        if (!relocate(idx, before, after, shared)) return POSTPONED;
    }
    common.resize(c);
    {
        const uint32_t u0 = us_index(grp[0]); const unsigned char* p0 = (const unsigned char*)seq_ptr(u0);
        const bool at_back = (cand.side == 0) != us_reverse(grp[0]);
        const Cursor first{at_back ? p0 + rec[u0].len - 1 : p0, at_back ? -1 : 1, us_reverse(grp[0]) ? g_lut.comp : g_lut.same};
        if (cand.side == 0) for (size_t i = 0; i < c; ++i) common[c - 1 - i] = (char)first.at(i);
        else for (size_t i = 0; i < c; ++i) common[i] = (char)first.at(i);
    }
    if (cand.side == 0) {   // shift_sequence_1 (:89-116): common end of the inputs moves to the start of this unitig
        for (uint32_t a = 0; a < gn; ++a) {
            const uint32_t s = us_index(grp[a]);
            if (!us_reverse(grp[a])) { rec[s].min_rpos += (uint32_t)c; rec[s].len -= (uint32_t)c; rec[s].room_after += (uint32_t)c; }                 // remove_seq_from_end, unitig.rs:225-232
            else { rec[s].min_fpos += (uint32_t)c; rec[s].len -= (uint32_t)c; rec[s].seq_off += c; rec[s].room_before += (uint32_t)c; }                // remove_seq_from_start, unitig.rs:216-223
        }
        // add_seq_to_start, unitig.rs:234-240
        rec[idx].seq_off -= c; rec[idx].room_before -= (uint32_t)c; rec[idx].len += (uint32_t)c; rec[idx].min_fpos -= (uint32_t)c;
        memcpy(arena + rec[idx].seq_off, common.data(), c);
    } else {                // shift_sequence_2 (:119-138): common start of the outputs moves to the end of this unitig
        for (uint32_t a = 0; a < gn; ++a) {
            const uint32_t s = us_index(grp[a]);
            if (!us_reverse(grp[a])) { rec[s].min_fpos += (uint32_t)c; rec[s].len -= (uint32_t)c; rec[s].seq_off += c; rec[s].room_before += (uint32_t)c; }
            else { rec[s].min_rpos += (uint32_t)c; rec[s].len -= (uint32_t)c; rec[s].room_after += (uint32_t)c; }
        }
        // add_seq_to_end, unitig.rs:242-248
        memcpy(arena + rec[idx].seq_off + rec[idx].len, common.data(), c);
        rec[idx].room_after -= (uint32_t)c; rec[idx].len += (uint32_t)c; rec[idx].min_rpos -= (uint32_t)c;
    }
    // Who has to look again?  (In the first pass every candidate after this one is still to come; only those already
    // visited need a mark.)  deps[u]: c[0]/c[1] read u's min_fpos/min_rpos; c[3],c[4] compare u's first bases, c[2],c[5] its
    // last bases.  A candidate that has nothing left in common ("exhausted") cannot be revived by a length or position
    // change, only by new bases at an end it compares (a "hard" mark).
    const int64_t below = first_pass ? (int64_t)ci : (int64_t)1 << 40;
    auto mark = [&](int32_t cnd, bool hard) {
        if (cnd < 0 || cnd >= below || (!hard && exhausted[cnd])) return;
        const uint64_t m = 1ull << (cnd & 63);
        if (shared) __atomic_fetch_or(&dirty[(size_t)cnd >> 6], m, __ATOMIC_RELAXED); else dirty[(size_t)cnd >> 6] |= m;
    };
    rec[idx].flags = pass_id;
    {
        const Deps& dd = deps[idx];      // the destination grew at its start (side 0) or end (side 1); its length changed
        const bool grew_start = cand.side == 0;
        mark(dd.c[3], grew_start); mark(dd.c[4], grew_start); mark(dd.c[2], !grew_start); mark(dd.c[5], !grew_start);
    }
    for (uint32_t a = 0; a < gn; ++a) {
        const uint32_t s = us_index(grp[a]);
        rec[s].flags = pass_id;
        const Deps& ds = deps[s];
        const bool trimmed_end = (cand.side == 0) != us_reverse(grp[a]);     // which physical end of s lost bases (its reader is this candidate)
        if (trimmed_end) { mark(ds.c[3], false); mark(ds.c[4], false); mark(ds.c[1], false); }   // readers of the other end see a new length; min_rpos moved
        else { mark(ds.c[2], false); mark(ds.c[5], false); mark(ds.c[0], false); }               // ... min_fpos moved
    }
    // A capped shift has to be looked at again in the next pass; after a complete one the bit must be off.
    if (c != common_len) { if (shared) __atomic_fetch_or(&dirty[w], bit_mask, __ATOMIC_RELAXED); else dirty[w] |= bit_mask; }
    return c;
}

// Passes in parallel.  Two candidates conflict when they share a unitig (destination or source); the reference's result only
// depends on the relative order of conflicting candidates.  Candidates are therefore levelled once (level = 1 + the highest
// level among earlier conflicting candidates) and every pass walks the levels in order, all threads applying the due
// candidates of one level at once: within a level no two candidates touch the same unitig.  A candidate marked during the
// pass conflicts with its marker, so it sits on another level: a later one if it comes later in the reference's order (then
// this pass still reaches it, as the reference's loop would), an earlier one otherwise (then it waits for the next pass).
// Shared writes: the work-list bits (atomic) and arena bumps (atomic; a candidate that finds the arena full is applied by one
// thread at the level's barrier, which is as good as any other place in its level).
void HostGraph::compute_levels() {
    // One serial sweep in candidate order; a byte per unitig keeps the table cache resident (beyond 250 levels the
    // passes are not worth their barriers and run as the plain sweep).
    const size_t n = cands.size();
    std::vector<uint8_t> level_of_unitig(U, 0), level(n);
    n_levels = 0;
    for (size_t ci = 0; ci < n; ++ci) {
        const Candidate& cd = cands[ci];
        const UStrand* grp = sources(cd);
        uint32_t lv = level_of_unitig[cd.idx];
        for (uint32_t a = 0; a < cd.gn; ++a) lv = std::max<uint32_t>(lv, level_of_unitig[us_index(grp[a])]);
        if (++lv > 250) { n_levels = 0xFFFFFFFFu; level_start.clear(); by_level.clear(); return; }
        level_of_unitig[cd.idx] = (uint8_t)lv;
        for (uint32_t a = 0; a < cd.gn; ++a) level_of_unitig[us_index(grp[a])] = (uint8_t)lv;
        level[ci] = (uint8_t)lv;
        if (lv > n_levels) n_levels = lv;
    }
    if (getenv("AC_HOST_PROFILE")) fprintf(stderr, "[host] expand levels %u for %zu candidates\n", n_levels, n);
    level_start.assign(n_levels + 2, 0); by_level.resize(n);
    for (size_t ci = 0; ci < n; ++ci) level_start[level[ci] + 1] += 1;
    for (uint32_t l = 1; l <= n_levels + 1; ++l) level_start[l] += level_start[l - 1];
    { std::vector<uint32_t> cur(level_start.begin(), level_start.end() - 1); for (size_t ci = 0; ci < n; ++ci) by_level[cur[level[ci]]++] = (uint32_t)ci; }
}

size_t HostGraph::pass_parallel(bool all_due) {
    static const bool tight = getenv("AC_EXPAND_TIGHT_ARENA") != nullptr;   // test hook: every relocation meets a full arena
    if (tight) arena_cap = arena_used;
    else if (all_due) {   // room for the relocations the first pass is known to need, so that (almost) nobody is handed back
        uint64_t reloc_bound = 0;
        for (size_t ci = 0; ci < cands.size(); ++ci)
            if (spec_len[ci] > AC_SEQ_SLACK) reloc_bound += (uint64_t)rec[cands[ci].idx].len + 2ull * spec_len[ci] + 8 * AC_SEQ_SLACK + 64;
        reserve_arena(reloc_bound);
    }
    const unsigned T = std::max<unsigned>(1, std::min<unsigned>(host_threads(), 16));
    std::vector<std::atomic<uint32_t>> next(n_levels + 2);
    for (auto& x : next) x.store(0);
    std::atomic<uint32_t> arrived{0}, generation{0};
    std::atomic<uint64_t> total{0}, evaluated{0};
    std::exception_ptr err = nullptr; std::atomic<bool> failed{false};
    std::mutex postponed_lock; std::vector<uint32_t> postponed;
    const uint32_t CHUNK = 128;
    struct Ctx { HostGraph* g; } ;
    auto work = [&]() {
        std::string common; uint64_t mine = 0, evals = 0;
        for (uint32_t l = 1; l <= n_levels; ++l) {
            const uint32_t lo = level_start[l], hi = level_start[l + 1];
            try {
                for (uint32_t c0; (c0 = next[l].fetch_add(CHUNK)) < hi - lo;) {
                    const uint32_t c1 = std::min(hi - lo, c0 + CHUNK);
                    for (uint32_t x = c0; x < c1; ++x) {
                        const uint32_t ci = by_level[lo + x];
                        if (!all_due) {
                            const uint64_t m = 1ull << (ci & 63);
                            if (!(__atomic_load_n(&dirty[ci >> 6], __ATOMIC_RELAXED) & m)) continue;
                            __atomic_fetch_and(&dirty[ci >> 6], ~m, __ATOMIC_RELAXED);
                        }
                        const size_t r = apply_candidate(ci, true, common);
                        ++evals;
                        if (r == POSTPONED) { std::lock_guard<std::mutex> lk(postponed_lock); postponed.push_back(ci); }
                        else mine += r;
                    }
                }
            } catch (...) { if (!failed.exchange(true)) err = std::current_exception(); }
            // barrier: nobody starts level l+1 before level l is complete; the last one in settles what was handed back
            const uint32_t gen = generation.load(std::memory_order_acquire);
            if (arrived.fetch_add(1, std::memory_order_acq_rel) + 1 == T) {
                try {
                    std::sort(postponed.begin(), postponed.end());
                    for (uint32_t ci : postponed) mine += apply_candidate(ci, false, common);
                } catch (...) { if (!failed.exchange(true)) err = std::current_exception(); }
                postponed.clear();
                arrived.store(0, std::memory_order_relaxed); generation.store(gen + 1, std::memory_order_release);
            } else {
                for (unsigned spins = 0; generation.load(std::memory_order_acquire) == gen; ++spins) { if (spins < 4096) __builtin_ia32_pause(); else std::this_thread::yield(); }
            }
        }
        total.fetch_add(mine); evaluated.fetch_add(evals);
    };
    run_on_threads(T, work);
    if (err) std::rethrow_exception(err);
    last_evaluations = (size_t)evaluated.load();
    return (size_t)total.load();
}

void HostGraph::prepare_simplify() {   // the structural part of expand_repeats: no sequence is read
    const double t0 = now_ms();
    if (!cands_ready) { compute_candidates(); prof.candidates = now_ms() - t0; }
}

// The lists compute_candidates() makes, taken from the device (pipeline.cu: CandidateFlagBody ... CommonLengthBody), which
// listed them in the numbering order it had just sorted.  Only valid for the graph exactly as built (a plain build).
bool HostGraph::adopt_candidates(const PipelineResult& r) {
    static const bool on_host = getenv("AC_HOST_CANDIDATES") != nullptr, cross_check = getenv("AC_CHECK_CANDIDATES") != nullptr;
    if (!r.cands || !r.deps || !r.fixed_start || on_host) return false;
    const double t0 = now_ms();
    if (cross_check) {                        // tests: the host listing of the same graph must agree field by field
        compute_candidates();
        bool same = cands.size() == r.n_cands && memcmp(fixed_start.data(), r.fixed_start, U) == 0 && memcmp(fixed_end.data(), r.fixed_end, U) == 0;
        for (size_t i = 0; same && i < cands.size(); ++i) {
            same = cands[i].idx == r.cands[i].idx && cands[i].side == r.cands[i].side && cands[i].gn == r.cands[i].gn && common_length(cands[i]) == r.spec_len[i];
            for (uint32_t a = 0; same && a < cands[i].gn; ++a) same = cands[i].src[a] == r.cands[i].src[a];
        }
        for (uint32_t u = 0; same && u < U; ++u) same = memcmp(&deps[u], &r.deps[u], sizeof(Deps)) == 0;
        if (!same) throw std::runtime_error("device and host candidate lists differ");
    }
    const size_t n = r.n_cands;
    const size_t T = std::max<size_t>(1, std::min<size_t>(host_threads(), (n + U) / 32768));
    cands.resize(n); deps.resize(U); spec_len.resize(n); spec_pass.resize(n); fixed_start.resize(U); fixed_end.resize(U);
    parallel_tasks(T, [&](size_t t) {
        const size_t a = n * t / T, b = n * (t + 1) / T, ua = (size_t)U * t / T, ub = (size_t)U * (t + 1) / T;
        if (b > a) { memcpy(&cands[a], r.cands + a, (b - a) * sizeof(Candidate)); memcpy(&spec_len[a], r.spec_len + a, (b - a) * 4); }
        if (ub > ua) { memcpy(&deps[ua], r.deps + ua, (ub - ua) * sizeof(Deps)); memcpy(&fixed_start[ua], r.fixed_start + ua, ub - ua); memcpy(&fixed_end[ua], r.fixed_end + ua, ub - ua); }
    });
    fixed_ready = true;
    compute_levels();
    dirty.assign((n + 63) / 64, 0);
    exhausted.assign(n, 0);
    first_pass = true; cands_ready = true; spec_from_device = true;
    prof.candidates = now_ms() - t0;
    return true;
}

size_t HostGraph::expand_repeats() {   // graph_simplification.rs:43-86
    const double t0 = now_ms();
    if (!cands_ready) { compute_candidates(); prof.candidates = now_ms() - t0; }
    size_t total_shifted = 0;
    ++pass_id;                                      // unitigs modified during this pass carry it in rec[].flags
    // the candidates known to be due (all of them in the first pass): compare their ends in parallel before they are applied
    std::vector<uint32_t> due;
    if (first_pass) { spec_len.resize(cands.size()); spec_pass.assign(cands.size(), 0); due.resize(cands.size()); for (size_t i = 0; i < due.size(); ++i) due[i] = (uint32_t)i; }
    else for (size_t w = 0; w < dirty.size(); ++w) for (uint64_t b = dirty[w]; b; b &= b - 1) due.push_back((uint32_t)(w * 64 + (size_t)__builtin_ctzll(b)));
    static const size_t min_due = getenv("AC_EXPAND_MIN_DUE") ? (size_t)atoll(getenv("AC_EXPAND_MIN_DUE")) : 2048;   // tests lower it to drive small graphs through the levels
    const bool parallel = due.size() >= min_due && host_threads() >= 4 && n_levels <= 250 && !getenv("AC_EXPAND_SERIAL");
    if (first_pass && spec_from_device) {         // compared on the device; the records were untouched since
        std::fill(spec_pass.begin(), spec_pass.end(), pass_id);
        spec_from_device = false;
    } else if (parallel || first_pass) {
        const size_t T = std::max<size_t>(1, std::min<size_t>(host_threads() * 4, due.size() / 512));
        parallel_tasks(T, [&](size_t t) {
            for (size_t x = due.size() * t / T; x < due.size() * (t + 1) / T; ++x) { spec_len[due[x]] = common_length(cands[due[x]]); spec_pass[due[x]] = pass_id; }
        });
    }
    if (first_pass) prof.compare = now_ms() - t0;
    if (parallel) { total_shifted = pass_parallel(first_pass); }
    else {
        std::string common;
        last_evaluations = 0;
        for (size_t w = 0; w < dirty.size() || (first_pass && w * 64 < cands.size()); ++w) {
            uint64_t passed = 0;                       // candidates of this word already visited in this pass
            for (;;) {
                // a candidate marked again at or behind the current position waits for the next pass, exactly as the
                // reference's loop would only reach it again in its next call
                const uint64_t avail = (first_pass ? ~0ull : dirty[w]) & ~passed;
                if (!avail) break;
                const int bit = __builtin_ctzll(avail);
                if (w * 64 + (size_t)bit >= cands.size()) break;
                passed = bit == 63 ? ~0ull : ((2ull << bit) - 1);
                if (!first_pass) dirty[w] &= ~(1ull << bit);
                total_shifted += apply_candidate(w * 64 + (size_t)bit, false, common); ++last_evaluations;
            }
        }
    }
    if (getenv("AC_HOST_PROFILE")) fprintf(stderr, "[host] pass %d%s: %zu evaluations, %zu bases, %.2f ms\n", prof.passes + 1, parallel ? " (by levels)" : "", last_evaluations, total_shifted, now_ms() - t0);
    first_pass = false;
    if (prof.passes == 0) prof.pass1 = now_ms() - t0;      // first pass (incl. candidate listing)
    prof.expand += now_ms() - t0; prof.passes += 1;
    return total_shifted;
}

void HostGraph::simplify_structure() {   // graph_simplification.rs:26-40
    while (expand_repeats() > 0) {}
    renumber();
    cands_ready = false;      // the numbering order changed: a later call starts from the new order
}

// ------------------------------------------------------------------------------------------------
// unitig_graph.rs:317-360 save_gfa
// ------------------------------------------------------------------------------------------------
namespace {
inline char* put_uint(char* p, uint64_t v) { auto r = std::to_chars(p, p + 24, v); return r.ptr; }
inline char* put_str(char* p, const char* s, size_t n) { memcpy(p, s, n); return p + n; }
inline uint32_t digits10(uint64_t v) { uint32_t d = 1; while (v >= 10) { v /= 10; ++d; } return d; }
// "{:.2}" of an f64 (unitig.rs:169): both Rust and printf render the exact binary value rounded half-to-even; only the
// spellings of the non-finite values differ.
inline uint32_t put_depth(char* p, double d) {
    if (d != d) { memcpy(p, "NaN", 3); return 3; }
    if (d - d != 0) { const bool neg = d < 0; memcpy(p, neg ? "-inf" : "inf", neg ? 4 : 3); return neg ? 4 : 3; }
    return (uint32_t)snprintf(p, 400, "%.2f", d);
}
const char* const COLOUR_TAG[4] = {"", "\tCL:Z:forestgreen", "\tCL:Z:pink", "\tCL:Z:steelblue"};   // unitig.rs:23-26, colour_tag :173-181 with use_other_colour = false
const char* const OTHER_COLOUR_TAG = "\tCL:Z:orangered";                                              // unitig.rs:27, use_other_colour = true
}  // namespace

uint32_t gfa_depth_text(char* p, double d) { return put_depth(p, d); }

void HostGraph::gfa_text(const std::vector<HostSeq>& seqs, std::string& out, bool other_colour) const {
    auto colour = [&](uint32_t idx) { const uint8_t t = type_of(idx); return t == 0 && other_colour ? OTHER_COLOUR_TAG : COLOUR_TAG[t]; };
    // Decimal text of every unitig number, by seed index, so that the hot loops copy bytes instead of dividing.
    std::vector<uint64_t> num_txt(U); std::vector<uint8_t> num_len(U);
    const size_t TU = std::max<size_t>(1, std::min<size_t>(host_threads() * 4, (size_t)U / 2048));
    auto ub = [&](size_t t) { return (uint32_t)((uint64_t)U * t / TU); };
    // task list: S-line blocks, L-line blocks (both by position in `order`), and P-line pieces (by path range)
    struct Piece { size_t seq; uint64_t a, b; };
    std::vector<Piece> pieces;
    const uint64_t P_CHUNK = 65536;
    for (size_t i = 0; i < seqs.size(); ++i) {
        uint64_t a = path_off[i];
        do { const uint64_t b = std::min(path_off[i + 1], a + P_CHUNK); pieces.push_back({i, a, b}); a = b; } while (a < path_off[i + 1]);
    }
    std::vector<uint64_t> s_size(TU), l_size(TU), p_size(pieces.size());
    parallel_tasks(TU, [&](size_t t) {
        for (uint32_t n = ub(t); n < ub(t + 1); ++n) {
            const uint32_t idx = order[n];
            if (number[idx] >= 100000000u) throw std::runtime_error("unitig numbers above 99,999,999 are not supported by the GFA writer");
            char buf[24]; const uint32_t d = (uint32_t)(put_uint(buf, (uint64_t)number[idx]) - buf);
            uint64_t v = 0; memcpy(&v, buf, d < 8 ? d : 8); num_txt[idx] = v; num_len[idx] = (uint8_t)d;
        }
    });
    parallel_tasks(TU, [&](size_t t) {
        uint64_t ss = 0, ls = 0;
        for (uint32_t n = ub(t); n < ub(t + 1); ++n) {
            const uint32_t idx = order[n];
            if (!depth_f) ss += 2 + num_len[idx] + 1 + rec[idx].len + 6 + digits10(depth[idx]) + 4;            // "S\t" num "\t" seq "\tDP:f:" depth ".00\n"
            else { char tmp[400]; ss += 2 + num_len[idx] + 1 + rec[idx].len + 6 + put_depth(tmp, depth_f[idx]) + strlen(colour(idx)) + 1; }
            for (uint32_t rev = 0; rev < 2; ++rev) {
                const UStrand from = us_make(idx, rev != 0);
                for (uint32_t x = next_off[from]; x < next_off[from + 1]; ++x)
                    ls += 2 + num_len[idx] + 3 + num_len[us_index(next[x])] + 2 + 4;           // "L\t" a "\t+\t" b "\t+" "\t0M\n"
            }
        }
        s_size[t] = ss; l_size[t] = ls;
    });
    parallel_tasks(pieces.size(), [&](size_t q) {
        const Piece& pc = pieces[q]; const HostSeq& s = seqs[pc.seq];
        uint64_t sz = 0;
        if (pc.a == path_off[pc.seq]) sz += 2 + digits10(s.id) + 1;                                                      // "P\t" id "\t"
        for (uint64_t x = pc.a; x < pc.b; ++x) sz += num_len[us_index(path[x])] + 2;                                  // num sign ","
        if (pc.b == path_off[pc.seq + 1]) {
            if (pc.b > pc.a) sz -= 1;                                                                                  // no comma after the last step
            sz += 8 + digits10(s.length) + 6 + s.filename.size() + 6 + s.contig_header.size() + 1;
            if (s.cluster > 0) sz += 6 + digits10(s.cluster);                                                          // "\tCL:i:" n (unitig_graph.rs:358)
        }
        p_size[q] = sz;
    });
    char head[64]; char* hp = put_str(head, "H\tVN:Z:1.0\tKM:i:", 16); hp = put_uint(hp, k); *hp++ = '\n';
    const uint64_t head_size = (uint64_t)(hp - head);
    std::vector<uint64_t> s_at(TU), l_at(TU), p_at(pieces.size());
    uint64_t at = head_size;
    for (size_t t = 0; t < TU; ++t) { s_at[t] = at; at += s_size[t]; }
    for (size_t t = 0; t < TU; ++t) { l_at[t] = at; at += l_size[t]; }
    for (size_t q = 0; q < pieces.size(); ++q) { p_at[q] = at; at += p_size[q]; }
    out.resize(at + 8);                 // 8 spare bytes: the number copies below write whole words
    char* const base = &out[0];
    memcpy(base, head, head_size);
    auto put_num = [&](char* p, uint32_t idx) { memcpy(p, &num_txt[idx], 8); return p + num_len[idx]; };

    parallel_tasks(2 * TU + pieces.size(), [&](size_t task) {
        if (task < TU) {                                        // S lines, unitig.rs:167-171; depth is integral so {:.2} renders as N.00
            char* p = base + s_at[task];
            for (uint32_t n = ub(task); n < ub(task + 1); ++n) {
                const uint32_t idx = order[n];
                *p++ = 'S'; *p++ = '\t'; p = put_uint(p, (uint64_t)number[idx]); *p++ = '\t';
                p = put_str(p, seq_ptr(idx), rec[idx].len);
                p = put_str(p, "\tDP:f:", 6);
                if (!depth_f) { p = put_uint(p, depth[idx]); p = put_str(p, ".00\n", 4); }
                else { char tmp[400]; const uint32_t dn = put_depth(tmp, depth_f[idx]); p = put_str(p, tmp, dn); const char* ct = colour(idx); p = put_str(p, ct, strlen(ct)); *p++ = '\n'; }
            }
            if ((uint64_t)(p - base) != s_at[task] + s_size[task]) throw std::runtime_error("GFA S-line size mismatch");
        } else if (task < 2 * TU) {                             // L lines, get_links_for_gfa :333-350: forward_next then reverse_next
            const size_t t = task - TU;
            char* p = base + l_at[t];
            for (uint32_t n = ub(t); n < ub(t + 1); ++n) {
                const uint32_t idx = order[n];
                for (uint32_t rev = 0; rev < 2; ++rev) {
                    const UStrand from = us_make(idx, rev != 0);
                    for (uint32_t x = next_off[from]; x < next_off[from + 1]; ++x) {
                        const UStrand to = next[x];
                        *p++ = 'L'; *p++ = '\t'; p = put_uint(p, (uint64_t)number[idx]); *p++ = '\t'; *p++ = rev ? '-' : '+'; *p++ = '\t';
                        p = put_uint(p, number[us_index(to)]); *p++ = '\t'; *p++ = us_reverse(to) ? '-' : '+'; p = put_str(p, "\t0M\n", 4);
                    }
                }
            }
            if ((uint64_t)(p - base) != l_at[t] + l_size[t]) throw std::runtime_error("GFA L-line size mismatch");
        } else {                                                // P lines, get_gfa_path_line :352-360
            const size_t q = task - 2 * TU;
            const Piece& pc = pieces[q]; const HostSeq& s = seqs[pc.seq];
            char* p = base + p_at[q];
            if (pc.a == path_off[pc.seq]) { *p++ = 'P'; *p++ = '\t'; p = put_uint(p, s.id); *p++ = '\t'; }
            const bool last_piece = pc.b == path_off[pc.seq + 1];
            for (uint64_t x = pc.a; x < pc.b; ++x) {
                // whole-word copies spill up to 7 bytes past the number; the spill is overwritten by this thread's next writes,
                // except near the end of the piece where the neighbouring piece may already be in place
                const uint32_t u = us_index(path[x]);
                if (x + 8 < pc.b) p = put_num(p, u); else { memcpy(p, &num_txt[u], num_len[u]); p += num_len[u]; }
                *p++ = us_reverse(path[x]) ? '-' : '+';
                if (!(last_piece && x + 1 == pc.b)) *p++ = ',';
            }
            if (last_piece) {
                p = put_str(p, "\t*\tLN:i:", 8); p = put_uint(p, s.length);
                p = put_str(p, "\tFN:Z:", 6); p = put_str(p, s.filename.data(), s.filename.size());
                p = put_str(p, "\tHD:Z:", 6); p = put_str(p, s.contig_header.data(), s.contig_header.size());
                if (s.cluster > 0) { p = put_str(p, "\tCL:i:", 6); p = put_uint(p, s.cluster); }
                *p++ = '\n';
            }
            if ((uint64_t)(p - base) != p_at[q] + p_size[q]) throw std::runtime_error("GFA P-line size mismatch");
        }
    });
    out.resize(at);
}
