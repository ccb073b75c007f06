// Device part of `autocycler cluster`: the contig distances (cluster.rs:132-192) and the UPGMA tree (cluster.rs:395-480).  This file
// compiles with nvcc for sm_90a (product) and with g++ -DAC_EMULATE (tests/emu: the bodies serially, UPGMA as a host loop).
#include "commands.h"

#include <cmath>
#include <string>

// ---- contig distances (cluster.rs:132-151): which sequences pass through each unitig, then every pair of them shares its length ----
struct PathMemberBody {
    const UStrand* path; const uint64_t* path_off; uint32_t n_seqs, words; uint32_t* member;
    AC_D void operator()(uint64_t x) const {
        uint32_t lo = 0, hi = n_seqs;                    // the sequence whose path holds step x
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (path_off[mid] <= x) lo = mid; else hi = mid; }
        ac_atomic_or(&member[(size_t)(path[x] >> 1) * words + (lo >> 5)], 1u << (lo & 31));
    }
};
struct PairShareBody {
    const uint32_t* member; const uint32_t* unitig_len; uint32_t n_seqs, words; unsigned long long* shared;
    AC_D void operator()(uint64_t u) const {
        const uint32_t* m = member + (size_t)u * words;
        const unsigned long long len = unitig_len[u];
        for (uint32_t wa = 0; wa < words; ++wa)
            for (uint32_t ba = m[wa]; ba; ba &= ba - 1) {
                const uint32_t a = (wa << 5) + (uint32_t)ac_ctz(ba);
                for (uint32_t wb = 0; wb < words; ++wb)
                    for (uint32_t bb = m[wb]; bb; bb &= bb - 1)
                        ac_atomic_add(&shared[(size_t)a * n_seqs + (wb << 5) + (uint32_t)ac_ctz(bb)], len);
            }
    }
};
// cluster.rs:145-149 and 177-192: the asymmetric distance 1 - shared / a_len (a_len: the u32 sum the reference converts) and its symmetric
// max.  No multiply, so nothing contracts into an FMA, and f64 division is IEEE: the bits equal ac_pairwise_distances' host division.
struct DistanceBody {
    const unsigned long long* shared; uint32_t n; double* asym; double* sym;
    AC_D void operator()(uint64_t x) const {
        const uint64_t a = x / n, b = x % n;
        const double d_ab = 1.0 - ((double)shared[x] / (double)(uint32_t)shared[a * n + a]);
        const double d_ba = 1.0 - ((double)shared[b * n + a] / (double)(uint32_t)shared[b * n + b]);
        asym[x] = d_ab;
        sym[x] = (d_ab != d_ab || d_ab < d_ba) ? d_ba : d_ab;       // f64::max: a NaN loses
    }
};

// ---- cluster: UPGMA (cluster.rs:395-480), see DESIGN.md §12 ----
// Clusters are indexed by their smallest member in ascending id order, so a merge of a < b keeps index a (new_id = a.min(b)).  The n x n
// working matrix M holds, above the diagonal, the mean distance D(i, j) of clusters i < j and, below it, their sum T(i, j) over all member
// pairs; T(a u b, j) = T(a, j) + T(b, j) and D = T / (|a u b| |j|).  Every live row i keeps its least (D, j) over j > i.
#define AC_UPGMA_NONE 0xFFFFFFFFu
// get_closest_pair (:461-480) scans pairs (a, b) in ascending id order with a strict <: the least (distance, a, b) wins
AC_HD bool upgma_less(double d1, uint32_t a1, uint32_t b1, double d2, uint32_t a2, uint32_t b2) {
    return d1 < d2 || (d1 == d2 && (a1 < a2 || (a1 == a2 && b1 < b2)));
}
// least live (D(i, j), j) over j = from, from + step, ... < n, folded into (bd, bj)
AC_HD void upgma_row_scan(const double* M, uint32_t n, const uint8_t* alive, uint32_t i, uint32_t from, uint32_t step, double& bd, uint32_t& bj) {
    for (uint32_t j = from; j < n; j += step)
        if (alive[j]) { const double d = M[(size_t)i * n + j]; if (upgma_less(d, i, j, bd, i, bj)) { bd = d; bj = j; } }
}
// cluster b has joined a (|a u b| = cnt_ab): the sum and the mean of (a u b, j)
AC_HD void upgma_merge_entry(double* M, uint32_t n, uint32_t a, uint32_t b, uint32_t j, uint64_t cnt_ab, uint64_t cnt_j) {
    double* t_a = j < a ? M + (size_t)a * n + j : M + (size_t)j * n + a;
    const double t_b = j < b ? M[(size_t)b * n + j] : M[(size_t)j * n + b];
    const double t = *t_a + t_b;
    *t_a = t;
    (j < a ? M[(size_t)j * n + a] : M[(size_t)a * n + j]) = t / (double)(cnt_ab * cnt_j);
}
// row i != a of a live cluster i < b after that merge: true when its minimum pointed at a or b and the row must be scanned again;
// otherwise the minimum stands, unless the new D(i, a) undercuts it
AC_HD bool upgma_row_after_merge(const double* M, uint32_t n, uint32_t a, uint32_t b, uint32_t i, double& rd, uint32_t& rj) {
    if (rj == a || rj == b) return true;
    if (i < a) { const double d = M[(size_t)i * n + a]; if (upgma_less(d, i, a, rd, i, rj)) { rd = d; rj = a; } }
    return false;
}

#ifndef AC_EMULATE
__device__ __forceinline__ void upgma_warp_min(double& d, uint32_t& a, uint32_t& b) {
    for (int o = 16; o; o >>= 1) {
        const double od = __shfl_down_sync(0xFFFFFFFFu, d, o);
        const uint32_t oa = __shfl_down_sync(0xFFFFFFFFu, a, o), ob = __shfl_down_sync(0xFFFFFFFFu, b, o);
        if (upgma_less(od, oa, ob, d, a, b)) { d = od; a = oa; b = ob; }
    }
}
// One persistent CTA performs all n - 1 merges (no launch or grid barrier per merge).  Per merge: the least row minimum (block
// reduction), the merged row (a thread per column), the rows whose minimum involved a or b (listed), then a warp per listed row scans it.
__global__ void __launch_bounds__(1024) ac_upgma_kernel(double* M, uint32_t n, uint8_t* alive, uint32_t* cnt, uint32_t* node, double* rd, uint32_t* rj,
                                                        uint32_t* list, UpgmaMerge* out, uint32_t first_node, uint32_t* done) {
    __shared__ double s_d[32];
    __shared__ uint32_t s_a[32], s_b[32], s_n, s_pair[2];
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    for (uint32_t i = warp; i < n; i += 32) {
        double bd = INFINITY; uint32_t bi = i, bj = AC_UPGMA_NONE;
        upgma_row_scan(M, n, alive, i, i + 1 + lane, 32, bd, bj);
        upgma_warp_min(bd, bi, bj);
        if (lane == 0) { rd[i] = bd; rj[i] = bj; }
    }
    __syncthreads();
    for (uint32_t step = 0; step + 1 < n; ++step) {
        double bd = INFINITY; uint32_t ba = AC_UPGMA_NONE, bb = AC_UPGMA_NONE;
        for (uint32_t i = tid; i < n; i += blockDim.x)
            if (alive[i] && upgma_less(rd[i], i, rj[i], bd, ba, bb)) { bd = rd[i]; ba = i; bb = rj[i]; }
        upgma_warp_min(bd, ba, bb);
        if (lane == 0) { s_d[warp] = bd; s_a[warp] = ba; s_b[warp] = bb; }
        __syncthreads();
        if (warp == 0) {
            bd = s_d[lane]; ba = s_a[lane]; bb = s_b[lane];
            upgma_warp_min(bd, ba, bb);
            if (lane == 0 && bb == AC_UPGMA_NONE) { s_pair[0] = AC_UPGMA_NONE; *done = step; }   // no comparable pair left (NaN distances)
            else if (lane == 0) {
                UpgmaMerge m; m.node = first_node + step; m.left = node[ba]; m.right = node[bb]; m.pad = 0; m.dist = bd / 2.0;
                out[step] = m;
                alive[bb] = 0; cnt[ba] += cnt[bb]; node[ba] = m.node;
                s_pair[0] = ba; s_pair[1] = bb; s_n = 0;
            }
        }
        __syncthreads();
        const uint32_t a = s_pair[0], b = s_pair[1];
        if (a == AC_UPGMA_NONE) return;                  // the same value for every thread
        const uint64_t cab = cnt[a];
        for (uint32_t j = tid; j < n; j += blockDim.x)
            if (alive[j] && j != a) upgma_merge_entry(M, n, a, b, j, cab, cnt[j]);
        __syncthreads();
        for (uint32_t i = tid; i < b; i += blockDim.x) {
            if (!alive[i]) continue;
            double d = rd[i]; uint32_t j = rj[i];
            if (i == a || upgma_row_after_merge(M, n, a, b, i, d, j)) list[atomicAdd(&s_n, 1u)] = i;
            else if (j != rj[i]) { rd[i] = d; rj[i] = j; }
        }
        __syncthreads();
        const uint32_t L = s_n;
        for (uint32_t x = warp; x < L; x += 32) {
            const uint32_t i = list[x];
            double rbd = INFINITY; uint32_t ri = i, rbj = AC_UPGMA_NONE;
            upgma_row_scan(M, n, alive, i, i + 1 + lane, 32, rbd, rbj);
            upgma_warp_min(rbd, ri, rbj);
            if (lane == 0) { rd[i] = rbd; rj[i] = rbj; }
        }
        __syncthreads();
    }
    if (tid == 0) *done = n - 1;
}
#endif

void DeviceCluster::upload_paths(const UStrand* path, const uint64_t* path_off, uint32_t n, const uint32_t* unitig_len, uint32_t U) {
    AcStream* st = &ctx.stream;
    const uint64_t steps = path_off[n];
    const uint32_t words = (n + 31) / 32;
    d_path.ensure(steps * 4 + 4); d_path_off.ensure(((size_t)n + 1) * 8); d_len.ensure((size_t)U * 4 + 4);
    member.ensure((size_t)U * words * 4 + 4); d_shared.ensure((size_t)n * n * 8);
    if (steps) ac_h2d(d_path.p, path, steps * 4, st);
    ac_h2d(d_path_off.p, path_off, ((size_t)n + 1) * 8, st);
    if (U) ac_h2d(d_len.p, unitig_len, (size_t)U * 4, st);
    ac_memset(member.p, 0, (size_t)U * words * 4 + 4, st);
    ac_memset(d_shared.p, 0, (size_t)n * n * 8, st);
}
void DeviceCluster::share_lengths(uint64_t steps, uint32_t n, uint32_t U) {
    const uint32_t words = (n + 31) / 32;
    ac_launch("path_member", &ctx.stream, PathMemberBody{d_path.as<UStrand>(), d_path_off.as<uint64_t>(), n, words, member.as<uint32_t>()}, steps);
    ac_launch("pair_share", &ctx.stream, PairShareBody{member.as<uint32_t>(), d_len.as<uint32_t>(), n, words, d_shared.as<unsigned long long>()}, U);
}

void DeviceCluster::pair_shared_lengths(const UStrand* path, const uint64_t* path_off, uint32_t n, const uint32_t* unitig_len, uint32_t U, uint64_t* shared) {
    ctx.make_current();
    if (n == 0) return;
    upload_paths(path, path_off, n, unitig_len, U);
    share_lengths(path_off[n], n, U);
    ac_d2h(shared, d_shared.p, (size_t)n * n * 8, &ctx.stream);
    ac_sync(&ctx.stream);
}

float DeviceCluster::cluster_distances(const UStrand* path, const uint64_t* path_off, uint32_t n, const uint32_t* unitig_len, uint32_t U, double* asym) {
    ctx.make_current();
    sym_n = 0;
    if (n == 0) return 0.f;
    const size_t nn = (size_t)n * n;
    d_asym.ensure(nn * 8); upgma_m.ensure(nn * 8);
    upload_paths(path, path_off, n, unitig_len, U);
    AcTimer timer(&ctx.stream);                               // the three kernels only: the uploads and memsets above are outside
    share_lengths(path_off[n], n, U);
    ac_launch("distance", &ctx.stream, DistanceBody{d_shared.as<unsigned long long>(), n, d_asym.as<double>(), upgma_m.as<double>()}, nn);
    timer.stop();
    ac_d2h(asym, d_asym.p, nn * 8, &ctx.stream);
    ac_sync(&ctx.stream);
    sym_n = n;
    return timer.ms();
}

float DeviceCluster::upgma(const double* sym, uint32_t n, const uint32_t* ids, UpgmaMerge* merges) {
    ctx.make_current();
    AcStream* st = &ctx.stream;
    for (uint32_t i = 1; i < n; ++i) if (ids[i] <= ids[i - 1]) throw std::runtime_error("upgma: ids must be strictly ascending");
    if (!sym && sym_n != n) throw std::runtime_error("upgma: no distance matrix of this size on the device");
    sym_n = 0;                                                // the kernel works in place
    if (n < 2) return 0.f;
    const size_t nn = (size_t)n * n;
    upgma_m.ensure(nn * 8); upgma_alive.ensure(n); upgma_cnt.ensure((size_t)n * 4); upgma_node.ensure((size_t)n * 4);
    upgma_rd.ensure((size_t)n * 8); upgma_rj.ensure((size_t)n * 4); upgma_list.ensure((size_t)n * 4); upgma_out.ensure((size_t)n * sizeof(UpgmaMerge));
    upgma_done.ensure(4);
    if (sym) ac_h2d(upgma_m.p, sym, nn * 8, st);
    const std::vector<uint32_t> ones(n, 1u);
    ac_memset(upgma_alive.p, 1, n, st);
    ac_h2d(upgma_cnt.p, ones.data(), (size_t)n * 4, st);
    ac_h2d(upgma_node.p, ids, (size_t)n * 4, st);
    double* M = upgma_m.as<double>(); uint8_t* alive = upgma_alive.as<uint8_t>(); uint32_t* cnt = upgma_cnt.as<uint32_t>(); uint32_t* node = upgma_node.as<uint32_t>();
    double* rd = upgma_rd.as<double>(); uint32_t* rj = upgma_rj.as<uint32_t>(); UpgmaMerge* out = upgma_out.as<UpgmaMerge>();
    const uint32_t first_node = ids[n - 1] + 1;
    AcTimer timer(st);
#ifndef AC_EMULATE
    ac_launch_kernel("upgma", st, ac_upgma_kernel, 1, 1024, 0, M, n, alive, cnt, node, rd, rj, upgma_list.as<uint32_t>(), out, first_node, upgma_done.as<uint32_t>());
#else
    // the kernel's steps, serially: row minima, least pair, merged row, then the rows that must be scanned again
    uint32_t& done_dev = *upgma_done.as<uint32_t>();
    for (uint32_t i = 0; i < n; ++i) { rd[i] = INFINITY; rj[i] = AC_UPGMA_NONE; upgma_row_scan(M, n, alive, i, i + 1, 1, rd[i], rj[i]); }
    done_dev = n - 1;
    for (uint32_t step = 0; step + 1 < n; ++step) {
        double bd = INFINITY; uint32_t a = AC_UPGMA_NONE, b = AC_UPGMA_NONE;
        for (uint32_t i = 0; i < n; ++i) if (alive[i] && upgma_less(rd[i], i, rj[i], bd, a, b)) { bd = rd[i]; a = i; b = rj[i]; }
        if (b == AC_UPGMA_NONE) { done_dev = step; break; }
        UpgmaMerge mg; mg.node = first_node + step; mg.left = node[a]; mg.right = node[b]; mg.pad = 0; mg.dist = bd / 2.0;
        out[step] = mg;
        alive[b] = 0; cnt[a] += cnt[b]; node[a] = mg.node;
        for (uint32_t j = 0; j < n; ++j) if (alive[j] && j != a) upgma_merge_entry(M, n, a, b, j, cnt[a], cnt[j]);
        for (uint32_t i = 0; i < b; ++i)
            if (alive[i] && (i == a || upgma_row_after_merge(M, n, a, b, i, rd[i], rj[i]))) {
                rd[i] = INFINITY; rj[i] = AC_UPGMA_NONE; upgma_row_scan(M, n, alive, i, i + 1, 1, rd[i], rj[i]);
            }
    }
#endif
    timer.stop();
    uint32_t done = 0;
    ac_d2h(merges, out, (size_t)(n - 1) * sizeof(UpgmaMerge), st);
    ac_d2h(&done, upgma_done.p, 4, st);
    ac_sync(st);
    if (done != n - 1) throw std::runtime_error("upgma: no pair of clusters with a comparable (non-NaN) distance is left after " + std::to_string(done) + " merges");
    return timer.ms();
}
