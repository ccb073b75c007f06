// Device part of `autocycler trim` (overlap alignments) and `autocycler resolve` (bridge path distances).  Both sweep one dynamic
// programming matrix per job by anti-diagonals, one CTA per job, with the three live diagonals in shared memory or in HBM scratch.  This
// file compiles with nvcc for sm_90a (product) and with g++ -DAC_EMULATE (tests/emu, a serial loop over the same cell functions).
#include "commands.h"

#include <algorithm>
#include <cmath>
#include <cstring>

// ------------------------------------------------------------------------------------------------
// trim: overlap alignment of unitig paths (trim.rs:366-479), see DESIGN.md §9
// ------------------------------------------------------------------------------------------------
// Every score is a sum of +w, -w and -(wi+wj)/2 with integral w < 2^32, so it is a multiple of 0.5 far below 2^52: f64 adds are exact
// and the matrix is the same in any evaluation order (the CTA's anti-diagonal sweep, the emulation's row-major loop, the reference's).
// The matrix itself is not kept: the traceback needs S[i-1][j] >= S[i][j-1] (:443) and path equality (:436), so the fill stores that
// one comparison per cell, packed 32 cells to a word along anti-diagonals (d = i + j); each diagonal starts on a word boundary.
#define AC_TRIM_GAP 0
#define AC_TRIM_NONE (-1)
AC_HD uint32_t trim_diag_lo(uint32_t d, uint32_t k) { return d > k ? d - k : 1u; }     // first row i of anti-diagonal d (2 <= d <= 2k)
AC_HD uint32_t trim_diag_words(uint32_t d, uint32_t k) {                             // 32-bit words of diagonal d's bits (0 outside 2..2k)
    if (d < 2 || d > 2 * k) return 0;
    const uint32_t hi = d - 1 < k ? d - 1 : k;
    return (hi - trim_diag_lo(d, k) + 1 + 31) / 32;
}
AC_HD uint64_t trim_bit_words(uint32_t k) { uint64_t w = 0; for (uint32_t d = 2; d <= 2 * k; ++d) w += trim_diag_words(d, k); return w; }
// :396-405, one cell: the diagonal, up (i-1, j) and left (i, j-1) scores, the two unitigs and their weights
AC_HD double trim_cell(double diag, double up, double left, int32_t a, int32_t b, double wa, double wb) {
    const double match_score = diag + (a == b ? wa : -(wa + wb) / 2.0);
    const double delete_score = up - wa, insert_score = left - wb;
    const double m = match_score > delete_score ? match_score : delete_score;      // f64::max without NaNs
    return m > insert_score ? m : insert_score;
}
// :413-419: the right edge S[i][k] is visited with i ascending and a strict > keeps the smallest i among ties
AC_HD void trim_edge(double s, uint32_t i, double& best, uint32_t& best_i) { if (s > best) { best = s; best_i = i; } }
// :431-461 from (max_i, k): writes the pieces in traceback order (last column first) and returns their count, or 0 when the walk ends
// on the left edge (i > 0).  pa = path_a (its first k entries are rows 1..k), pb = path_b + n - k (columns 1..k), bits as above.
AC_HD uint32_t trim_traceback(const int32_t* pa, const int32_t* pb, uint32_t n, uint32_t k, const uint32_t* bits, uint32_t max_i, AlignPiece* out) {
    uint32_t i = max_i, j = k, cnt = 0;
    uint64_t off = 0;
    for (uint32_t d = 2; d < i + j; ++d) off += trim_diag_words(d, k);
    while (i > 0 && j > 0) {
        const uint32_t d = i + j;
        const int32_t a = pa[i - 1], b = pb[j - 1];
        const int32_t gi = (int32_t)(i - 1), gj = (int32_t)(n - k + j - 1);
        if (a == b) {
            out[cnt++] = AlignPiece{a, gi, b, gj};
            --i; --j;
            off -= trim_diag_words(d - 1, k) + trim_diag_words(d - 2, k);
        } else {
            const uint32_t t = i - trim_diag_lo(d, k);
            if ((bits[off + t / 32] >> (t % 32)) & 1u) { out[cnt++] = AlignPiece{a, gi, AC_TRIM_GAP, AC_TRIM_NONE}; --i; }
            else { out[cnt++] = AlignPiece{AC_TRIM_GAP, AC_TRIM_NONE, b, gj}; --j; }
            off -= trim_diag_words(d - 1, k);
        }
    }
    return i > 0 ? 0 : cnt;
}
// Per job: where its bit words, its traceback output (2k pieces), and, for windows beyond shared memory, its three diagonals (HBM) live.
struct TrimLaunchJob { uint64_t a_off, b_off, bits_off, out_off, scratch_off; uint32_t n, k, skip, slot; };

#ifndef AC_EMULATE
// One CTA per job sweeps the 2k-1 anti-diagonals; the three live ones (d-2, d-1, d, indexed by row i) sit in shared memory, or in the
// job's HBM scratch when 24 (k + 1) bytes exceed the CTA's shared memory (same code, another base pointer).  A thread owns a cell per
// 1024 of its diagonal: the two path entries it reads are adjacent to its neighbours' (coalesced), and its warp packs the 32 traceback
// bits with one ballot into one word.  Thread 0 then runs the O(k) traceback over those bits.
__global__ void __launch_bounds__(1024) ac_overlap_align_kernel(const TrimLaunchJob* __restrict__ jobs, const int32_t* __restrict__ values,
                                                                const uint32_t* __restrict__ weights, uint32_t* __restrict__ bits,
                                                                double* scratch, AlignPiece* __restrict__ out, uint32_t* __restrict__ out_len, int use_shared) {
    extern __shared__ double trim_smem[];
    __shared__ double best;
    __shared__ uint32_t best_i;
    const TrimLaunchJob J = jobs[blockIdx.x];
    const uint32_t k = J.k, tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    double* D = use_shared ? trim_smem : scratch + J.scratch_off;
    const int32_t* pa = values + J.a_off;
    const int32_t* pb = values + J.b_off + (J.n - k);
    uint32_t* B = bits + J.bits_off;
    const uint32_t diag_shift = J.n - k;             // global_i == global_j  <=>  i - 1 == n - k + j - 1
    if (tid == 0) { best = -INFINITY; best_i = 0; }
    uint64_t off = 0;
    for (uint32_t d = 2; d <= 2 * k; ++d) {
        double* cur = D + (size_t)(d % 3) * (k + 1);
        const double* prev = D + (size_t)((d - 1) % 3) * (k + 1);
        const double* prev2 = D + (size_t)((d - 2) % 3) * (k + 1);
        const uint32_t lo = trim_diag_lo(d, k), hi = d - 1 < k ? d - 1 : k, len = hi - lo + 1;
        for (uint32_t base = 0; base < len; base += blockDim.x) {      // the same trip count for every thread: all lanes reach the ballot
            const uint32_t t = base + tid;
            bool up_wins = false;
            if (t < len) {
                const uint32_t i = lo + t, j = d - i;
                const double up = i == 1 ? 0.0 : prev[i - 1];
                const double left = j == 1 ? 0.0 : prev[i];
                up_wins = up >= left;
                double s = -INFINITY;
                if (!(J.skip && i == j + diag_shift)) {
                    const double diag = (i == 1 || j == 1) ? 0.0 : prev2[i - 1];
                    const int32_t a = pa[i - 1], b = pb[j - 1];
                    s = trim_cell(diag, up, left, a, b, (double)__ldg(weights + (a < 0 ? -a : a)), (double)__ldg(weights + (b < 0 ? -b : b)));
                }
                cur[i] = s;
                if (j == k) trim_edge(s, i, best, best_i);         // one cell per diagonal, rows in ascending order
            }
            const uint32_t word = __ballot_sync(0xFFFFFFFFu, up_wins);
            if (lane == 0 && base + warp * 32 < len) B[off + base / 32 + warp] = word;
        }
        off += (len + 31) / 32;
        __syncthreads();
    }
    if (tid == 0) {
        AlignPiece* o = out + J.out_off;
        out_len[J.slot] = best > 0.0 ? trim_traceback(pa, pb, J.n, k, B, best_i, o) : 0;      // :422 max_score <= 0: no alignment
    }
}
#endif

// ------------------------------------------------------------------------------------------------
// resolve: all-pairs path distances of a bridge (global_alignment_distance, resolve.rs:387-418), see DESIGN.md §13
// ------------------------------------------------------------------------------------------------
// D[i][j] over rows i (the shorter path a) and columns j (path b), in u32 with wraparound as the reference's release build computes it.
// The sweep goes by anti-diagonals d = i + j; the three live ones (d-2, d-1, d) are indexed by row i, n + 1 words each.  Swapping the
// two paths transposes the recurrence and applies the same adds and mins to the same operands, so D(a, b) == D(b, a) bit for bit.
#define AC_BRIDGE_THREADS 256
AC_HD uint32_t bridge_weight(const uint32_t* w, int32_t u) { return w[u < 0 ? (uint32_t)(-(int64_t)u) : (uint32_t)u]; }
// One cell (i, j = d - i) of diagonal d from the two diagonals before it: the top edge (gaps in a), the left edge (gaps in b), or the
// min of match/mismatch, delete and insert (:404-411).
AC_HD void bridge_cell(uint32_t* cur, const uint32_t* prev, const uint32_t* prev2, uint32_t i, uint32_t j, const int32_t* pa, const int32_t* pb,
                       const uint32_t* w) {
    if (i == 0) { cur[0] = prev[0] + bridge_weight(w, pb[j - 1]); return; }
    const int32_t a = pa[i - 1];
    const uint32_t wa = bridge_weight(w, a);
    if (j == 0) { cur[i] = prev[i - 1] + wa; return; }
    const int32_t b = pb[j - 1];
    const uint32_t wb = bridge_weight(w, b);
    const uint32_t match_or_mismatch = prev2[i - 1] + (a == b ? 0u : (wa > wb ? wa : wb));
    const uint32_t delete_cost = prev[i - 1] + wa, insert_cost = prev[i] + wb;
    const uint32_t m = match_or_mismatch < delete_cost ? match_or_mismatch : delete_cost;
    cur[i] = m < insert_cost ? m : insert_cost;
}
AC_HD uint32_t bridge_diag_lo(uint32_t d, uint32_t m) { return d > m ? d - m : 0u; }
AC_HD uint32_t bridge_diag_hi(uint32_t d, uint32_t n) { return d < n ? d : n; }
// Per job: its two paths, where its diagonals live when they exceed shared memory, and its output slot.
struct BridgeLaunchJob { uint64_t a_off, b_off, scratch_off; uint32_t n, m, slot, pad; };

#ifndef AC_EMULATE
// One CTA per job.  The diagonals sit in dynamic shared memory, or in the job's HBM scratch when 12 (n + 1) bytes exceed the CTA's
// shared memory (same code, another base pointer).  Thread t owns rows t, t + 256, ... of every diagonal: neighbouring threads read
// neighbouring path entries and diagonal words.
__global__ void __launch_bounds__(AC_BRIDGE_THREADS) ac_bridge_distance_kernel(const BridgeLaunchJob* __restrict__ jobs, const int32_t* __restrict__ values,
                                                                               const uint32_t* __restrict__ weights, uint32_t* scratch,
                                                                               uint32_t* __restrict__ dist, int use_shared) {
    extern __shared__ uint32_t bridge_smem[];
    const BridgeLaunchJob J = jobs[blockIdx.x];
    const uint32_t n = J.n, m = J.m, stride = n + 1;
    uint32_t* D = use_shared ? bridge_smem : scratch + J.scratch_off;
    const int32_t* pa = values + J.a_off;
    const int32_t* pb = values + J.b_off;
    if (threadIdx.x == 0) D[0] = 0;                   // d = 0: D[0][0]
    __syncthreads();
    for (uint32_t d = 1; d <= n + m; ++d) {
        uint32_t* cur = D + (size_t)(d % 3) * stride;
        const uint32_t* prev = D + (size_t)((d - 1) % 3) * stride;
        const uint32_t* prev2 = D + (size_t)((d + 1) % 3) * stride;     // d - 2 (mod 3); not read on d = 1
        const uint32_t hi = bridge_diag_hi(d, n);
        for (uint32_t i = bridge_diag_lo(d, m) + threadIdx.x; i <= hi; i += AC_BRIDGE_THREADS) bridge_cell(cur, prev, prev2, i, d - i, pa, pb, weights);
        __syncthreads();
    }
    if (threadIdx.x == 0) dist[J.slot] = D[(size_t)((n + m) % 3) * stride + n];
}
#endif

// ------------------------------------------------------------------------------------------------
// host side, shared by both: one CTA per job, largest first (the long sweeps start before the short ones), the jobs whose three live
// diagonals fit one CTA's shared memory in one launch and those that keep them in HBM scratch in a second
// ------------------------------------------------------------------------------------------------
static uint32_t overlap_shared_k_max() { return (uint32_t)((ac_smem_optin() - 64) / 24) - 1; }   // 24 (k + 1) bytes beside 64 B of static shared variables
static uint32_t bridge_shared_n_max() { return (uint32_t)(ac_smem_optin() / 12) - 1; }          // 12 (n + 1) bytes; no static shared variables

// Puts the jobs in launch order (by size, descending; the shared-memory ones first) and gives every HBM job 3 (rows + 1) cells of
// scratch.  Returns the number of shared-memory jobs; max_rows: the largest row count among them, scratch: the cells handed out.
template <class Job, class Rows, class Size>
static uint32_t plan_jobs(std::vector<Job>& lj, uint32_t shared_rows, Rows rows, Size size, uint32_t& max_rows, uint64_t& scratch) {
    std::stable_sort(lj.begin(), lj.end(), [&](const Job& a, const Job& b) { return size(a) > size(b); });
    std::stable_partition(lj.begin(), lj.end(), [&](const Job& L) { return rows(L) <= shared_rows; });
    uint32_t n_shared = 0;
    max_rows = 0; scratch = 0;
    for (Job& L : lj) {
        if (rows(L) <= shared_rows) { ++n_shared; max_rows = std::max(max_rows, rows(L)); }
        else { L.scratch_off = scratch; scratch += 3ull * (rows(L) + 1); }
    }
    return n_shared;
}

#ifndef AC_EMULATE
// The two launches over the planned jobs: the shared-memory ones with smem bytes of dynamic shared memory, then the HBM ones.  The
// kernel's arguments are (jobs, args..., use_shared).
template <class Kernel, class Job, class... A>
static void launch_jobs(const char* name, const char* name_hbm, AcStream* st, Kernel kernel, unsigned threads, size_t smem, const Job* jobs,
                        uint32_t n_jobs, uint32_t n_shared, A... args) {
    if (n_shared) ac_launch_kernel(name, st, kernel, n_shared, threads, smem, jobs, args..., 1);
    if (n_shared < n_jobs) ac_launch_kernel(name_hbm, st, kernel, n_jobs - n_shared, threads, 0, jobs + n_shared, args..., 0);
}
#endif

static void check_weights(const int32_t* values, uint64_t n_values, uint64_t n_weights, const char* what) {
    for (uint64_t v = 0; v < n_values; ++v) {
        const int64_t a = values[v] < 0 ? -(int64_t)values[v] : values[v];
        if ((uint64_t)a >= n_weights) throw std::runtime_error(std::string(what) + ": unitig without a weight");
    }
}

float DeviceAlign::overlap_align(const int32_t* values, uint64_t n_values, const uint32_t* weights, uint64_t n_weights,
                                 const OverlapJob* jobs, uint32_t n_jobs, std::vector<std::vector<AlignPiece>>& out, AlignRun* run_info) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    out.assign(n_jobs, {});
    if (run_info) *run_info = AlignRun();
    const uint32_t shared_k = overlap_shared_k_max();
    std::vector<uint32_t> run;                       // windows of k = 0 have no cell
    for (uint32_t x = 0; x < n_jobs; ++x) {
        if (jobs[x].k > jobs[x].n) throw std::runtime_error("overlap_align: window larger than the path");
        if (jobs[x].k > 0) run.push_back(x);
    }
    if (run.empty()) return 0.f;
    std::vector<TrimLaunchJob> lj(run.size());
    uint64_t bits_words = 0, out_pieces = 0;
    for (size_t r = 0; r < run.size(); ++r) {
        const OverlapJob& J = jobs[run[r]];
        if (J.a_off + J.n > n_values || J.b_off + J.n > n_values) throw std::runtime_error("overlap_align: path outside the value array");
        TrimLaunchJob& L = lj[r];
        L.a_off = J.a_off; L.b_off = J.b_off; L.n = J.n; L.k = J.k; L.skip = J.skip_diagonal ? 1 : 0; L.slot = (uint32_t)r;
        L.bits_off = bits_words; bits_words += trim_bit_words(J.k);
        L.out_off = out_pieces; out_pieces += 2ull * J.k;
        L.scratch_off = 0;
    }
    uint32_t k_shared = 0; uint64_t scratch = 0;
    const auto rows = [](const TrimLaunchJob& L) { return L.k; };
    const uint32_t n_shared = plan_jobs(lj, shared_k, rows, rows, k_shared, scratch);
    if (run_info) {
        run_info->shared_jobs = n_shared; run_info->hbm_jobs = (uint32_t)lj.size() - n_shared;
        run_info->buffer_bytes = lj.size() * sizeof(TrimLaunchJob) + n_values * 4 + n_weights * 4 + bits_words * 4 + out_pieces * sizeof(AlignPiece) +
                                 run.size() * 4 + scratch * 8;
    }
    trim_jobs.ensure(lj.size() * sizeof(TrimLaunchJob)); trim_vals.ensure(n_values * 4 + 4); trim_w.ensure(n_weights * 4 + 4);
    trim_bits.ensure(bits_words * 4 + 4); trim_out.ensure(out_pieces * sizeof(AlignPiece) + 16); trim_len.ensure(run.size() * 4);
    trim_scratch.ensure(scratch * 8 + 8);
    ac_h2d(trim_jobs.p, lj.data(), lj.size() * sizeof(TrimLaunchJob), st);
    if (n_values) ac_h2d(trim_vals.p, values, n_values * 4, st);
    if (n_weights) ac_h2d(trim_w.p, weights, n_weights * 4, st);
    check_weights(values, n_values, n_weights, "overlap_align");
    std::vector<uint32_t> len(run.size());
    AcTimer timer(st);
#ifndef AC_EMULATE
    launch_jobs("overlap_align", "overlap_align_hbm", st, ac_overlap_align_kernel, 1024, (size_t)24 * (k_shared + 1), trim_jobs.as<TrimLaunchJob>(),
                (uint32_t)lj.size(), n_shared, trim_vals.as<int32_t>(), trim_w.as<uint32_t>(), trim_bits.as<uint32_t>(), trim_scratch.as<double>(),
                trim_out.as<AlignPiece>(), trim_len.as<uint32_t>());
#else
    // the same per-cell recurrence, right-edge maximum and traceback, in row-major order (a topological order of the matrix)
    (void)n_shared;
    uint32_t* bits = trim_bits.as<uint32_t>();
    memset(bits, 0, bits_words * 4);
    for (const TrimLaunchJob& L : lj) {
        const uint32_t k = L.k;
        const int32_t* pa = trim_vals.as<int32_t>() + L.a_off;
        const int32_t* pb = trim_vals.as<int32_t>() + L.b_off + (L.n - k);
        const uint32_t* w = trim_w.as<uint32_t>();
        std::vector<uint64_t> diag_off(2 * (size_t)k + 2, 0);
        for (uint32_t d = 3; d <= 2 * k + 1; ++d) diag_off[d] = diag_off[d - 1] + trim_diag_words(d - 1, k);
        std::vector<double> above(k + 1, 0.0), row(k + 1, 0.0);
        double best = -INFINITY; uint32_t best_i = 0;
        for (uint32_t i = 1; i <= k; ++i) {
            row[0] = 0.0;
            for (uint32_t j = 1; j <= k; ++j) {
                const double up = above[j], left = row[j - 1];
                const uint32_t d = i + j, t = i - trim_diag_lo(d, k);
                if (up >= left) bits[L.bits_off + diag_off[d] + t / 32] |= 1u << (t % 32);
                double s = -INFINITY;
                if (!(L.skip && i == j + (L.n - k))) {
                    const int32_t a = pa[i - 1], b = pb[j - 1];
                    s = trim_cell(above[j - 1], up, left, a, b, (double)w[a < 0 ? -a : a], (double)w[b < 0 ? -b : b]);
                }
                row[j] = s;
            }
            trim_edge(row[k], i, best, best_i);
            above.swap(row);
        }
        trim_len.as<uint32_t>()[L.slot] = best > 0.0 ? trim_traceback(pa, pb, L.n, k, bits + L.bits_off, best_i, trim_out.as<AlignPiece>() + L.out_off) : 0;
    }
#endif
    timer.stop();
    ac_d2h(len.data(), trim_len.p, run.size() * 4, st);
    ac_sync(st);
    // the pieces of every job sit at the front of its 2k slots, last column first
    for (const TrimLaunchJob& L : lj) {
        if (!len[L.slot]) continue;
        std::vector<AlignPiece>& o = out[run[L.slot]];
        o.resize(len[L.slot]);
        ac_d2h(o.data(), trim_out.as<AlignPiece>() + L.out_off, (size_t)len[L.slot] * sizeof(AlignPiece), st);
    }
    ac_sync(st);
    for (auto& o : out) std::reverse(o.begin(), o.end());
    return timer.ms();
}

float DeviceAlign::bridge_distances(const int32_t* values, uint64_t n_values, const uint32_t* weights, uint64_t n_weights,
                                    const BridgeJob* jobs, uint32_t n_jobs, uint32_t* dist, AlignRun* run_info) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    if (run_info) *run_info = AlignRun();
    if (n_jobs == 0) return 0.f;
    check_weights(values, n_values, n_weights, "bridge_distances");
    const uint32_t shared_n = bridge_shared_n_max();
    std::vector<BridgeLaunchJob> lj(n_jobs);
    for (uint32_t x = 0; x < n_jobs; ++x) {
        const BridgeJob& J = jobs[x];
        if (J.n > J.m) throw std::runtime_error("bridge_distances: the rows must be the shorter path");
        if (J.a_off + J.n > n_values || J.b_off + J.m > n_values) throw std::runtime_error("bridge_distances: path outside the value array");
        lj[x] = BridgeLaunchJob{J.a_off, J.b_off, 0, J.n, J.m, x, 0};
    }
    uint32_t n_max_shared = 0; uint64_t scratch = 0;
    const uint32_t n_shared = plan_jobs(lj, shared_n, [](const BridgeLaunchJob& L) { return L.n; },
                                        [](const BridgeLaunchJob& L) { return (uint64_t)L.n * L.m; }, n_max_shared, scratch);
    if (run_info) {
        run_info->shared_jobs = n_shared; run_info->hbm_jobs = n_jobs - n_shared;
        run_info->buffer_bytes = lj.size() * sizeof(BridgeLaunchJob) + n_values * 4 + n_weights * 4 + scratch * 4 + (uint64_t)n_jobs * 4;
    }
    br_jobs.ensure(lj.size() * sizeof(BridgeLaunchJob)); br_vals.ensure(n_values * 4 + 4); br_w.ensure(n_weights * 4 + 4);
    br_scratch.ensure(scratch * 4 + 4); br_dist.ensure((size_t)n_jobs * 4);
    ac_h2d(br_jobs.p, lj.data(), lj.size() * sizeof(BridgeLaunchJob), st);
    if (n_values) ac_h2d(br_vals.p, values, n_values * 4, st);
    if (n_weights) ac_h2d(br_w.p, weights, n_weights * 4, st);
    AcTimer timer(st);
#ifndef AC_EMULATE
    launch_jobs("bridge_distance", "bridge_distance_hbm", st, ac_bridge_distance_kernel, AC_BRIDGE_THREADS, (size_t)12 * (n_max_shared + 1),
                br_jobs.as<BridgeLaunchJob>(), n_jobs, n_shared, br_vals.as<int32_t>(), br_w.as<uint32_t>(), br_scratch.as<uint32_t>(), br_dist.as<uint32_t>());
#else
    // the same diagonals and per-cell body, one job and one cell at a time
    const int32_t* vals = br_vals.as<int32_t>();
    const uint32_t* w = br_w.as<uint32_t>();
    std::vector<uint32_t> own;
    for (const BridgeLaunchJob& L : lj) {
        const uint32_t stride = L.n + 1;
        uint32_t* D;
        if (L.n <= shared_n) { own.assign(3 * (size_t)stride, 0xA5A5A5A5u); D = own.data(); }
        else D = br_scratch.as<uint32_t>() + L.scratch_off;
        D[0] = 0;
        for (uint32_t d = 1; d <= L.n + L.m; ++d) {
            uint32_t* cur = D + (size_t)(d % 3) * stride;
            const uint32_t* prev = D + (size_t)((d - 1) % 3) * stride;
            const uint32_t* prev2 = D + (size_t)((d + 1) % 3) * stride;
            for (uint32_t i = bridge_diag_lo(d, L.m); i <= bridge_diag_hi(d, L.n); ++i) bridge_cell(cur, prev, prev2, i, d - i, vals + L.a_off, vals + L.b_off, w);
        }
        br_dist.as<uint32_t>()[L.slot] = D[(size_t)((L.n + L.m) % 3) * stride + L.n];
    }
#endif
    timer.stop();
    ac_d2h(dist, br_dist.p, (size_t)n_jobs * 4, st);
    ac_sync(st);
    return timer.ms();
}
