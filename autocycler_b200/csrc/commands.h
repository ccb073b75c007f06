// The device parts of `autocycler trim`, `resolve`, `cluster`, `dotplot`, `subsample`, `helper genome_size`, `depth`, `qv`, `unassembled`,
// `polish` and `variants`.  Each object owns its device buffers (allocated on first use, kept for the next call) and runs on the device and stream
// of the DeviceContext it is given, which must outlive it.
#pragma once
#include <cstdint>
#include <functional>
#include <vector>

#include "backend.h"
#include "pipeline.h"

// One overlap alignment of `autocycler trim` (trim.rs:366-479): path_a's first k entries against path_b's last k, k = min(max_unitigs, n).
// Both paths are n signed unitig numbers in the caller's value array.  skip_diagonal: the start-end form (path_a == path_b, cells with
// global_i == global_j stay -inf, :395).
struct OverlapJob { uint64_t a_off, b_off; uint32_t n, k, skip_diagonal, pad; };
// One column of the traceback (trim.rs:329-335): GAP = 0 as a unitig, NONE = -1 as an index.
struct AlignPiece { int32_t a_unitig, a_index, b_unitig, b_index; };
// One path distance of `autocycler resolve` (global_alignment_distance, resolve.rs:387-418): the n values at a_off (rows, the shorter
// path) against the m values at b_off, signed unitig numbers in the caller's value array.
struct BridgeJob { uint64_t a_off, b_off; uint32_t n, m; };
// What one overlap_align or bridge_distances call ran: jobs whose live diagonals sat in shared memory, jobs whose diagonals sat in HBM
// scratch (one launch for each form that has jobs), and the device buffer bytes the call planned for its jobs, paths, weights, scratch
// and outputs.
struct AlignRun {
    uint32_t shared_jobs = 0, hbm_jobs = 0;
    uint64_t buffer_bytes = 0;
    uint32_t launches() const { return (shared_jobs > 0) + (hbm_jobs > 0); }
};

// What a batch of trim or resolve clusters ran on the device, over all its overlap_align or bridge_distances calls: clusters, kernel
// launches, jobs, DP cells, the largest call's planned buffer bytes and the kernels' time (CUDA events; 0 under emulation).
struct AlignBatch {
    uint32_t clusters = 0, launches = 0;
    uint64_t jobs = 0, cells = 0, buffer_bytes = 0;
    float kernel_ms = 0.f;
};

// Trim's overlap alignments and resolve's bridge distances: one CTA per job sweeps the anti-diagonals, with the three live ones in
// shared memory or, when they do not fit, in HBM scratch.
class DeviceAlign {
public:
    explicit DeviceAlign(DeviceContext& ctx) : ctx(ctx) {}
    ~DeviceAlign() { ctx.make_current(); }
    // trim.rs overlap_alignment up to the traceback, for a batch of jobs: fill, right-edge maximum and traceback on the device.
    // weights[|unitig|] = unitig length.  out[j] = the traceback's pieces in alignment order, empty when the best right-edge score is <= 0
    // or the traceback ends on the left edge; the identity test is the caller's.  Returns the kernels' time in ms (0 under emulation).
    float overlap_align(const int32_t* values, uint64_t n_values, const uint32_t* weights, uint64_t n_weights,
                        const OverlapJob* jobs, uint32_t n_jobs, std::vector<std::vector<AlignPiece>>& out, AlignRun* run = nullptr);
    // resolve.rs:387-418 for a batch of path pairs: dist[x] = the u32 (wrapping) edit distance of job x, weights[|unitig|] = unitig
    // length.  Returns the kernels' time in ms (0 under emulation).
    float bridge_distances(const int32_t* values, uint64_t n_values, const uint32_t* weights, uint64_t n_weights,
                           const BridgeJob* jobs, uint32_t n_jobs, uint32_t* dist, AlignRun* run);
private:
    DeviceContext& ctx;
    DevBuf trim_jobs, trim_vals, trim_w, trim_bits, trim_scratch, trim_out, trim_len;
    DevBuf br_jobs, br_vals, br_w, br_scratch, br_dist;
};

// One merge of `autocycler cluster`'s UPGMA (cluster.rs:410-430): the new node's number, its left child (the cluster with the smaller
// id), its right child, and the node's distance to the tips (half the merged pair's mean distance).
struct UpgmaMerge { uint32_t node, left, right, pad; double dist; };

class DeviceCluster {
public:
    explicit DeviceCluster(DeviceContext& ctx) : ctx(ctx) {}
    ~DeviceCluster() { ctx.make_current(); }
    // cluster.rs:132-151 pairwise_contig_distances, the integer part: shared[a * n_seqs + b] = total length of the unitigs that the
    // paths of sequences a and b have in common (the diagonal is the length of a's own unitig set).  Host arrays in, host array out.
    void pair_shared_lengths(const UStrand* path, const uint64_t* path_off, uint32_t n_seqs, const uint32_t* unitig_len, uint32_t n_unitigs, uint64_t* shared);
    // cluster.rs:132-192: the same shared lengths turned into the asymmetric distance matrix on the device (copied back into
    // asym[n_seqs * n_seqs]) and its symmetric max, which stays in HBM for upgma(nullptr, ...).  Returns the kernels' time in ms.
    float cluster_distances(const UStrand* path, const uint64_t* path_off, uint32_t n_seqs, const uint32_t* unitig_len, uint32_t n_unitigs, double* asym);
    // UPGMA (cluster.rs:395-480) in one persistent CTA: n - 1 merges of the n clusters ids[0..n) (strictly ascending), new nodes numbered
    // from ids[n-1] + 1.  sym: a symmetric n x n host matrix, or null for the one cluster_distances left on the device (used up).
    // Returns the kernel's time in ms (0 under emulation).
    float upgma(const double* sym, uint32_t n, const uint32_t* ids, UpgmaMerge* merges);
private:
    void upload_paths(const UStrand* path, const uint64_t* path_off, uint32_t n, const uint32_t* unitig_len, uint32_t U);   // and clears the outputs
    void share_lengths(uint64_t steps, uint32_t n, uint32_t U);
    DeviceContext& ctx;
    DevBuf d_path, d_path_off, d_len, member, d_shared, d_asym;      // the paths and lengths of the call, not the compress graph's
    DevBuf upgma_m, upgma_alive, upgma_cnt, upgma_node, upgma_rd, upgma_rj, upgma_list, upgma_out, upgma_done;
    uint32_t sym_n = 0;                                      // upgma_m holds cluster_distances' symmetric matrix of this many sequences (0: none)
};

// One sequence of `autocycler dotplot` (dotplot.rs:394-450): its bytes at off in the caller's byte array, its first window's global
// index (ascending; a sequence shorter than k has no windows) and the pixel its box starts at.
struct DotplotSeq { uint64_t off, window_base; uint32_t len, start_px; };
// What one dotplot call ran: windows with only ACGT (the device's), their distinct canonical k-mers, dots (sum of the groups' squared
// sizes) and the kernels' time in ms (CUDA events; 0 under emulation).
struct DotplotRun { uint64_t windows = 0, groups = 0, dots = 0; float kernel_ms = 0.f; };

// A dot's key (dotplot.rs:202-211 loop order, last writer wins): the pixel shows the dot with the largest (a * n + b, j, forward), so
// the key packs the pair of sequences above bit 34, b's window j in bits 2-33, forward in bit 1, and bit 0 set (0 is "no dot").
inline uint64_t dotplot_key(uint64_t pair, uint32_t j, bool forward) { return (pair << 34) | ((uint64_t)j << 2) | ((uint64_t)forward << 1) | 1u; }
#define AC_DOTPLOT_MAX_SEQS 32768u    // n * n pairs fit the key's 30 pair bits
#define AC_DOT_SCAN_TILE 32           // values per thread of the u64 scan

class DeviceDotplot {
public:
    explicit DeviceDotplot(DeviceContext& ctx) : ctx(ctx) {}
    ~DeviceDotplot() { ctx.make_current(); }
    // dotplot.rs:202-211 for every ordered pair of sequences at once: each window of only ACGT is grouped with the windows that share its
    // canonical k-mer, and each ordered pair of windows in a group is one dot at (pixel of the first, pixel of the second), pixel =
    // start_px + round(position / bpp).  Every pixel keeps the largest dot key (dotplot_key); host_idx / host_key add the dots the host
    // found for the windows that hold other bytes.  rgb (res x res x 3) holds the base image on entry and the image with the dots on
    // return.  bytes: the sequences, uppercased, at seqs[s].off.
    void dotplot(const uint8_t* bytes, uint64_t n_bytes, const DotplotSeq* seqs, uint32_t n_seqs, uint32_t k, double bpp, uint32_t res,
                 const uint64_t* host_idx, const uint64_t* host_key, uint64_t n_host, uint8_t* rgb, DotplotRun* run);
private:
    template <int W> void windows(uint64_t N, uint32_t n_seqs, uint32_t k, double bpp, uint64_t mask);
    DeviceContext& ctx;
    DeviceScan scan;
    SerialScan<uint64_t, AC_DOT_SCAN_TILE, 8> scan_u64;          // of the groups' dot counts
    DevBuf d_bytes, d_seqs, d_keys, d_px, d_tag, d_rep, d_cnt, d_off, d_fill, d_gpx, d_gtag, d_table, d_gstart, d_gsize, d_gdots, d_pix, d_rgb, d_hidx, d_hkey;
};

// One FASTQ record of `autocycler subsample` in its window: where its header, sequence and quality start (the '@', the line ends and
// a trailing '\r' left out) and their lengths; the quality has seq_len bytes.
struct SubRecord { uint64_t head, seq, qual; uint32_t head_len, seq_len; };
// Why a record is refused, in the order the record body checks.  A window's first refused record is kept as (record << 3) | reason.
enum SubReason : uint32_t { SUB_NO_AT = 1, SUB_NO_PLUS = 2, SUB_TRUNCATED = 3, SUB_UNEQUAL = 4, SUB_TOO_LONG = 5 };
#define AC_SUB_NONE64 0xFFFFFFFFFFFFFFFFull
// What one window scan found: complete records (every record when the window ends the file), the bytes they span (the next window
// starts there) and the first refused record (AC_SUB_NONE64: none).
struct SubScan { uint64_t records = 0, cut = 0, bad = AC_SUB_NONE64; };
// One subset's rows of the statistics: count, bases, and the ascending n50 (metrics.rs:44-62).
struct SubStats { uint64_t count = 0, bases = 0, n50 = 0; };
#define AC_SUB_SCAN_TILE 32          // values per thread of the u64 scans (histogram rows, output offsets)

class DeviceSubsample {
public:
    explicit DeviceSubsample(DeviceContext& ctx) : ctx(ctx) {}
    ~DeviceSubsample() { ctx.make_current(); }
    // Pass 1 over one window of n bytes of FASTQ text (host memory; eof: the window ends the file).  Finds its complete records (at eof,
    // every record, the last one possibly without its newline), checks them and appends their sequence lengths to the file-wide length
    // array at `first` when keep_lengths.  The records stay on the device for gather() until the next scan.
    SubScan scan_window(const uint8_t* bytes, uint64_t n, bool eof, uint64_t first, bool keep_lengths);
    // The input's statistics over the first n lengths.
    SubStats input_stats(uint64_t n);
    // rank[order[p]] = p for the shuffled read order (n reads).
    void set_order(const uint32_t* order, uint64_t n);
    // Every subset's statistics at once: read r is in subset i when (rank[r] - starts[i]) mod n < rps.
    void subset_stats(uint64_t n, const uint64_t* starts, uint32_t count, uint64_t rps, SubStats* out);
    // Pass 2 for the window last scanned (its first record `first`): subset (start, rps)'s records, each as `@head\nseq\n+\nqual\n`, in
    // input order, into host_out (window bytes + 1 fit).  Returns the bytes written.
    uint64_t gather(uint64_t first, uint64_t n, uint64_t start, uint64_t rps, uint8_t* host_out);
    // Pinned host memory for the windows and the gathered output, kept with the device buffers.
    PinBuf h_win, h_out;
    float kernel_ms = 0.f;           // the kernels of every call so far (CUDA events; 0 under emulation)
    double copy_ms = 0.0;            // host wall time of the window uploads and the gathered output's copies back
    // The window last scanned, on the device: its bytes and its records' spans (valid until the next scan_window).
    const uint8_t* window_bytes() { return d_bytes.as<uint8_t>(); }
    const SubRecord* window_records() { return d_rec.as<SubRecord>(); }
private:
    void rows(uint64_t n, const uint64_t* starts, uint32_t count, uint64_t rps, SubStats* out);
    DeviceContext& ctx;
    DeviceScan scan;
    SerialScan<uint64_t, AC_SUB_SCAN_TILE, 8> scan_u64;
    uint64_t win_records = 0, win_bytes = 0;
    DevBuf d_bytes, d_mask, d_cnt, d_line, d_rec, d_bad, d_len, d_len_tmp, d_rank, d_starts, d_h1, d_s1, d_h2, d_s2, d_row, d_size, d_out;
};

// `autocycler helper genome_size`: the canonical k-mer depth spectrum of a FASTQ file (DESIGN.md §18).  Each window that
// DeviceSubsample scanned is packed into a device-resident stream (2 bits and a validity bit per base, every record from a fresh
// 32-base word); the k-mers are then counted in P partitions of an open-addressing table of 16-byte slots, and each partition's counts
// are added to a histogram of AC_GS_BINS bins (the last one holds every count >= AC_GS_BINS - 1).
#define AC_GS_BINS 16384u
struct GsSlot { uint64_t key; uint32_t count, pad; };   // key: canonical k-mer + 1 (0: empty)
// What the count ran: partitions, the largest table's bytes, partitions rerun with twice the slots, and the kernels' time by stage.
struct SpectrumRun { uint64_t partitions = 0, table_bytes = 0, reruns = 0; float pack_ms = 0.f, count_ms = 0.f, hist_ms = 0.f; };

class DeviceSpectrum {
public:
    explicit DeviceSpectrum(DeviceContext& ctx) : ctx(ctx) {}
    ~DeviceSpectrum() { ctx.make_current(); }
    // An empty packed stream for k-mers of length k (odd, 11..31).
    void begin(uint32_t k);
    // Appends the `records` records of the window `sub` scanned last to the packed stream, and adds their windows and bases.
    void pack_window(DeviceSubsample& sub, uint64_t records);
    // W: windows of k valid bases inside one read, and the bases of the records packed so far (one host round trip).
    void totals(uint64_t* windows, uint64_t* bases);
    // The histogram of the packed stream's canonical k-mer counts into hist[AC_GS_BINS].  budget_slots: the most slots a table may
    // take; parts: the partitions to use (0: the smallest power of two whose 2 W / P slots fit the budget).  A partition whose probe
    // limit is hit is counted again with twice the slots.
    void count(uint64_t windows, uint64_t budget_slots, uint64_t parts, uint64_t* hist, SpectrumRun* run);
    // A further sweep over the partitions count() made, for a rule that needs the whole histogram first: each(table, slots, P, part) runs
    // once per partition with that partition's table on the device.  The table the last count or sweep left behind goes first (after
    // count(), the last partition's); every other partition is counted again at the slots count() settled on (run gets those counts'
    // time, and any rerun).  With one partition a sweep counts nothing.
    void sweep(const std::function<void(const GsSlot*, uint64_t, uint64_t, uint64_t)>& each, SpectrumRun* run);
    float kernel_ms = 0.f;           // the kernels of every call since begin() (CUDA events; 0 under emulation)
    // The packed stream so far, on the device: `packed_words()` words of codes and validity masks (DeviceDepth::probe reads it).
    const uint64_t* packed_codes() { return d_code.as<uint64_t>(); }
    const uint32_t* packed_valid() { return d_valid.as<uint32_t>(); }
    uint64_t packed_words() const { return words; }
    float packed_ms() const { return pack_ms; }      // the packing's kernels since begin()
    // The last pack_window's records' first words, relative to the words packed before it, and their total (records + 1 values).
    const uint64_t* window_word_offsets() { return d_woff.as<uint64_t>(); }
private:
    uint64_t count_partition(uint64_t parts, uint64_t part, uint64_t slots, SpectrumRun* run);
    DeviceContext& ctx;
    SerialScan<uint64_t, AC_SUB_SCAN_TILE, 8> scan_u64;          // of the records' word counts
    uint32_t k = 21;
    uint64_t words = 0;              // packed words so far
    uint64_t resident = 0;           // the partition whose table d_table holds
    float pack_ms = 0.f;
    std::vector<uint64_t> part_slots;                            // each partition's slots in the last count()
    DevBuf d_code, d_valid, d_woff, d_tot, d_table, d_flag, d_hist;
};
// Slots of device memory a k-mer table may take by default: half of the device's free memory (2^25 slots under emulation).
uint64_t ac_gs_budget_slots();

// `autocycler depth`: each contig's read depth from the reads' canonical k-mers (DESIGN.md §19).  The contigs are packed like the reads
// (DeviceSpectrum's layout, each contig from a fresh word) and every window's canonical key goes into one open-addressing table; a key
// seen twice is marked non-unique.  The reads' packed stream then probes the table, each hit on a unique key adding 1 to its count, and
// each contig's depth is the exact median of its unique keys' counts, selected on the device.
struct DepthSlot { uint64_t key; uint32_t count, flags; };   // key: canonical k-mer + 1 (0: empty); flags: contig id, AC_DEPTH_DUP
#define AC_DEPTH_DUP 0x80000000u                             // the key occurs more than once over the assembly's windows
// What the device ran: the assembly's windows, the table's bytes and the kernels' time by stage (CUDA events; 0 under emulation).
struct DepthRun { uint64_t assembly_windows = 0, table_bytes = 0; float pack_ms = 0.f, insert_ms = 0.f, probe_ms = 0.f, median_ms = 0.f; };

class DeviceDepth {
public:
    explicit DeviceDepth(DeviceContext& ctx) : ctx(ctx) {}
    ~DeviceDepth() { ctx.make_current(); }
    // The assembly table.  bytes: every contig's bytes back to back (a circular contig followed by its first k-1 bases), contig c
    // taking len[c] of them; windows: the windows of k A/C/G/T bases in them.  The table takes max(2 windows, 64) slots;
    // std::length_error when that exceeds budget_slots or there are 2^31 contigs or more.
    void build(const uint8_t* bytes, const uint64_t* len, uint32_t n_contigs, uint64_t windows, uint32_t k, uint64_t budget_slots, DepthRun* run);
    // Counts every window of the reads `spec` packed (after build, with the same k) into the unique keys it hits.
    void probe(DeviceSpectrum& spec, DepthRun* run);
    // unique[c]: contig c's unique keys; median[c]: the median of their counts (NaN when unique[c] is 0).  Host arrays of n_contigs.
    void medians(uint64_t* unique, double* median, DepthRun* run);
private:
    DeviceContext& ctx;
    uint32_t k = 21, n_contigs = 0;
    uint64_t slots = 0;
    DevBuf d_bytes, d_contig, d_woff, d_code, d_valid, d_wcid, d_table, d_unique, d_rank, d_prefix, d_hist, d_median;
};

// `autocycler qv`: each assembly's k-mer accuracy and completeness against the reads (DESIGN.md §20).  Every assembly's contigs are packed
// into one stream (depth's layout) and their canonical keys claimed in one combined DepthSlot table with the flags left 0, so the reads'
// packed stream, probed once with DpProbeBody, counts every hit.  Then, per assembly, a multiplicity table of its own keys (each with the
// reads' count copied from the combined table), a mask of its unsupported windows, and its copy-number spectrum.
struct QvSlot { uint64_t key; uint32_t m, r; };              // key: canonical k-mer + 1 (0: empty); m: the assembly's windows; r: the reads'
#define AC_QV_CN 5                                           // copy-number columns of the spectrum: m = 0 (unused on the device), 1, 2, 3, 4+
// What the device ran: every assembly's windows, the two tables' bytes and the kernels' time by stage (CUDA events; 0 under emulation).
struct QvRun { uint64_t assembly_windows = 0, table_bytes = 0; float pack_ms = 0.f, insert_ms = 0.f, probe_ms = 0.f, assembly_ms = 0.f; };

class DeviceQv {
public:
    explicit DeviceQv(DeviceContext& ctx) : ctx(ctx) {}
    ~DeviceQv() { ctx.make_current(); }
    // The combined table and the per-assembly buffers.  bytes: every contig's bytes back to back (a circular contig followed by its first
    // k-1 bases), contig c taking len[c] of them; assembly a holds contigs first[a] .. first[a+1]-1 and windows[a] windows of k A/C/G/T
    // bases.  The combined table takes max(2 sum windows, 64) slots, the multiplicity table max(2 max windows, 64); std::length_error when
    // the two exceed budget_slots.
    void build(const uint8_t* bytes, const uint64_t* len, uint32_t n_contigs, const uint32_t* first, uint32_t n_assemblies,
               const uint64_t* windows, uint32_t k, uint64_t budget_slots, QvRun* run);
    // Counts every window of the reads `spec` packed (after build, with the same k) into the assembly key it hits.
    void probe(DeviceSpectrum& spec, QvRun* run);
    // Assembly a against the threshold t: mask[i] (one u32 per packed word of its contigs, from contig first[a]'s first word) has bit j
    // set when the window that ends at base j of that word has a read count below t; spectrum[c * AC_QV_CN + m] (AC_GS_BINS rows) counts
    // its distinct keys with read count bin c (min(r, AC_GS_BINS - 1)) that occur m times (4: 4 or more) over its windows.
    void assembly(uint32_t a, uint32_t t, uint32_t* mask, uint32_t* spectrum, QvRun* run);
    // The first packed word of every contig, and one past the last (n_contigs + 1 values), as build laid them out.
    const std::vector<uint64_t>& word_offsets() const { return woff; }
private:
    DeviceContext& ctx;
    uint32_t k = 21;
    uint64_t slots = 0, mult_slots = 0;
    std::vector<uint64_t> woff, win;
    std::vector<uint32_t> first_contig;
    DevBuf d_bytes, d_contig, d_code, d_valid, d_wcid, d_table, d_mult, d_mask, d_spec;
};

// `autocycler unassembled`: the reads an assembly does not explain (DESIGN.md §21).  The contigs of every input are packed (depth's
// layout) and their canonical keys claimed in one DepthSlot table, the assembly set A.  While the reads are packed, each packed word gets
// its read's index and each read its length.  After DeviceSpectrum::count has given the histogram and so the solid threshold t, a second
// sweep over its partitions counts, per read, the windows whose key the reads hold t times or more (s) and those of them A does not hold
// (a), and bins the distinct such keys that A does not hold by their read count.
// What the device ran: the assembly's windows, the bytes of the assembly set, the per-read counters and the word indices, and the
// kernels' time by stage (CUDA events; 0 under emulation).  sweep: the second sweep's recounts of partitions.
struct UaRun {
    uint64_t assembly_windows = 0, table_bytes = 0, read_bytes = 0;
    float pack_ms = 0.f, claim_ms = 0.f, index_ms = 0.f, attribute_ms = 0.f;
    SpectrumRun sweep;
};

class DeviceUnassembled {
public:
    explicit DeviceUnassembled(DeviceContext& ctx) : ctx(ctx) {}
    ~DeviceUnassembled() { ctx.make_current(); }
    // The assembly set.  bytes: every contig's bytes back to back (a circular contig followed by its first k-1 bases), contig c taking
    // len[c] of them, `windows` windows of k A/C/G/T bases in all.  The table takes max(2 windows, 64) slots; std::length_error when that
    // exceeds budget_slots.
    void build(const uint8_t* bytes, const uint64_t* len, uint32_t n_contigs, uint64_t windows, uint32_t k, uint64_t budget_slots, UaRun* run);
    // After spec.pack_window of the window whose first record is `first` and which has `records` records, starting at packed word `word0`:
    // each of its packed words gets its read's index, and each read its sequence length.
    void index_window(DeviceSpectrum& spec, DeviceSubsample& sub, uint64_t first, uint64_t records, uint64_t word0, UaRun* run);
    // The counters of `reads` reads and the word indices, with the assembly set, against budget_slots (16-byte slots); std::length_error
    // when they exceed it.
    void check_budget(uint64_t reads, uint64_t words, uint64_t budget_slots, UaRun* run);
    // After spec.count: the second sweep at threshold t.  counts[2 i] = s_i and counts[2 i + 1] = a_i for each of the `reads` reads,
    // lengths[i] its sequence length, absent[c] the distinct keys with bin(r) = c (r >= t) that A does not hold (host arrays).
    void attribute(DeviceSpectrum& spec, uint64_t reads, uint32_t t, uint32_t* counts, uint32_t* lengths, uint64_t* absent, UaRun* run);
private:
    DeviceContext& ctx;
    uint32_t k = 21;
    uint64_t slots = 0;
    DevBuf d_bytes, d_contig, d_code, d_valid, d_wcid, d_table, d_read, d_len, d_counts, d_absent;
};

// `autocycler polish`: the consensus corrected where the reads' k-mers do not support it (DESIGN.md §22).  Each round packs the contigs
// (depth's layout) and claims their canonical keys in a DepthSlot query table; a sweep over the read spectrum's partitions copies each
// key's read count r into the table, and a mask of the windows with r < t goes back to the host, which builds the loci.  For every
// attempted locus and each of its candidate edits, the k + s windows of the edited sequence that cover the edit are claimed in a candidate
// table, filled by a second sweep, and scored by their minimum r; one warp per locus then picks the best score and counts the candidates
// that hold it.
struct PlLocus { uint64_t word0, len, a; uint32_t circular, pad; };   // its contig's first packed word and length; the first unsupported window
// Candidate c of a locus at a largest indel of L (cur: the round's base at p0, 0..3 for A, C, G, T): the bases it puts at p0 (base i in
// bits 2i..2i+1, mlen of them) and the round's bases from p0 on that they replace (skip).  0..2: the other three bases in A, C, G, T
// order; 3..L+2: deletion of c-2 bases; then the insertions of 1, 2, ... L bases, each length's strings in lexicographic order.
struct PlEdit { uint32_t mid, mlen, skip; };
AC_HD PlEdit pl_edit(uint32_t c, uint32_t L, uint32_t cur) {
    if (c < 3) return PlEdit{c < cur ? c : c + 1, 1, 1};
    if (c < 3 + L) return PlEdit{0, 0, c - 2};
    uint32_t i = c - 3 - L, s = 1, n = 4;
    while (i >= n) { i -= n; ++s; n *= 4; }
    uint32_t mid = 0;
    for (uint32_t j = 0; j < s; ++j) mid |= ((i >> (2 * (s - 1 - j))) & 3u) << (2 * j);
    return PlEdit{mid, s, 0};
}
// What the device ran: the window table's bytes, the largest candidate table's, the candidate batches, and the kernels' time by stage
// (CUDA events; 0 under emulation).  sweep: the sweeps' recounts of partitions (none with one partition).
struct PlRun {
    uint64_t table_bytes = 0, candidate_bytes = 0, batches = 0;
    float pack_ms = 0.f, fill_ms = 0.f, candidate_ms = 0.f, choose_ms = 0.f;
    SpectrumRun sweep;
};

class DevicePolish {
public:
    explicit DevicePolish(DeviceContext& ctx) : ctx(ctx) {}
    ~DevicePolish() { ctx.make_current(); }
    // The candidates per locus at a largest indel of L (3 + L + sum_{s=1..L} 4^s) and their checked windows (sum of k + s).
    static uint64_t candidates(uint32_t max_indel);
    static uint64_t candidate_windows(uint32_t k, uint32_t max_indel);
    // The buffers for every round, before the read spectrum takes its share of the device: contigs of up to `bytes` bytes (junction bases
    // included) in `words` packed words with `windows` windows.  The window table takes max(2 windows, 64) slots; std::length_error when
    // that exceeds budget_slots.
    void reserve(uint64_t bytes, uint64_t words, uint64_t windows, uint32_t k, uint64_t budget_slots, PlRun* run);
    // One round's contigs (after reserve, within its sizes; after spec.count with the same k): bytes back to back, contig c taking len[c]
    // of them (a circular contig followed by its first k-1 bases).  mask[i] (one u32 per packed word, each contig from a fresh word) has
    // bit j set when the window that ends at base j of that word has a read count below t.
    void windows(DeviceSpectrum& spec, const uint8_t* bytes, const uint64_t* len, uint32_t n_contigs, uint64_t windows, uint32_t t, uint32_t* mask,
                 PlRun* run);
    // The candidates of n loci of the round windows() packed last, in batches whose candidate tables fit budget_slots (std::length_error
    // when one locus's does not).  out[3 i .. 3 i + 2] = locus i's best score (0: no candidate passes), the candidates that hold it and
    // the first of them.
    void choose(DeviceSpectrum& spec, const PlLocus* loci, uint64_t n, uint32_t max_indel, uint32_t t, uint64_t budget_slots, uint32_t* out,
                PlRun* run);
    // windows()'s first steps: the contigs packed and their keys claimed in the query table, with every count 0 (fill it in a sweep).
    void pack(const uint8_t* bytes, const uint64_t* len, uint32_t n_contigs, uint64_t windows, PlRun* run);
    // choose()'s claim, fill and score of the candidates of n loci, batch by batch: each(first locus, loci, device scores) runs after a
    // batch's scores (score[i * C + c], as PlScoreBody writes them) are on the device's stream.
    void score(DeviceSpectrum& spec, const PlLocus* loci, uint64_t n, uint32_t max_indel, uint32_t t, uint64_t budget_slots,
               const std::function<void(uint64_t, uint64_t, const uint32_t*)>& each, PlRun* run);
    // The round packed last, on the device: its codes, validity masks and packed words, and the query table of its keys.
    const uint64_t* packed_codes() { return d_code.as<uint64_t>(); }
    const uint32_t* packed_valid() { return d_valid.as<uint32_t>(); }
    uint64_t packed_words() const { return words; }
    DepthSlot* query_table() { return d_table.as<DepthSlot>(); }
    uint64_t query_slots() const { return slots; }
    uint32_t kmer() const { return k; }
private:
    void fill(DeviceSpectrum& spec, DepthSlot* table, uint64_t slots, PlRun* run);
    DeviceContext& ctx;
    uint32_t k = 21;
    uint64_t slots = 0, words = 0;
    DevBuf d_bytes, d_contig, d_code, d_valid, d_wcid, d_table, d_mask, d_loci, d_cand, d_score, d_out;
};

// `autocycler variants`: the alleles the reads carry beside the consensus (DESIGN.md §23).  The input is packed and its keys claimed and
// filled as polish's first round (DevicePolish::pack and a sweep of PlFillBody); in the same sweep VaScreenBody looks up, for the window
// that ends at each base p, the three windows S(p, b) with the last base swapped, and sets a bit where r >= t.  The host turns the masks
// into candidates, DevicePolish::score scores them, and VaRefBody gives each passing candidate the input's ref count and PK.
// One candidate to measure: its position as a polish locus (a = p - k + 1) and its index in pl_edit's order.
struct VaCandidate { PlLocus lo; uint32_t c, pad; };
// What the device ran beyond the polish object's steps: the screen's and the ref pass's time (CUDA events; 0 under emulation).
struct VaRun { float screen_ms = 0.f, ref_ms = 0.f; };

class DeviceVariants {
public:
    explicit DeviceVariants(DeviceContext& ctx) : ctx(ctx) {}
    ~DeviceVariants() { ctx.make_current(); }
    // After pl.pack: one sweep over the spectrum's partitions fills pl's query table and screens every window.  mask[3 w + j] (host, three
    // u32 per packed word) has bit i set when the window ending at base i of word w, its last base replaced by the j-th of the other three
    // bases in A, C, G, T order, has r >= t.
    void screen(DeviceSpectrum& spec, DevicePolish& pl, uint32_t t, uint32_t* mask, PlRun* prun, VaRun* run);
    // pl.score for n loci of the input: score[i * C + c] (host) as PlScoreBody writes it, C = DevicePolish::candidates(max_indel).
    void scores(DeviceSpectrum& spec, DevicePolish& pl, const PlLocus* loci, uint64_t n, uint32_t max_indel, uint32_t t, uint64_t budget_slots,
                uint32_t* score, PlRun* prun);
    // out[2 i] = candidate i's ref (the least r over the input's windows that start at a .. p + d, 0 for a missing one) and out[2 i + 1] its
    // PK (checked windows whose key pl's query table holds, the last one left out for an indel).  Host arrays.
    void ref(DevicePolish& pl, const VaCandidate* cand, uint64_t n, uint32_t max_indel, uint32_t* out, VaRun* run);
private:
    DeviceContext& ctx;
    DevBuf d_mask, d_cand, d_out;
};
