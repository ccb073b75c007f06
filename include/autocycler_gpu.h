/* autocycler_gpu.h — C ABI of libautocycler_gpu.so, the H100 implementation of Autocycler's
 * `compress` hot path.
 *
 * The reference (rrwick/Autocycler v0.6.1, Rust) has no FFI for this path; the path sits behind
 * in-crate calls.  Each entry point below names the reference interface it replaces (file:line
 * under the reference's src/), so that a Rust `extern "C"` shim (INTEGRATION.md) can bind them in
 * place of those calls:
 *
 *   KmerGraph::new + add_sequences          kmer_graph.rs:79-90      -> ac_create, ac_add_sequence, ac_upload
 *   UnitigGraph::from_kmer_graph            unitig_graph.rs:36-48    -> ac_build
 *   (the UnitigGraph / Unitig fields)       unitig_graph.rs:28-33, unitig.rs:30-45 -> ac_counts_get, ac_unitigs_copy
 *   simplify_structure                      graph_simplification.rs:26-40 -> ac_simplify
 *   merge_linear_paths (downstream, 8f)     graph_simplification.rs:315-371 -> ac_merge_linear_paths
 *   UnitigGraph::save_gfa                   unitig_graph.rs:317-331  -> ac_gfa_size, ac_gfa_copy
 *   compress (the whole subcommand)         compress.rs:32-50        -> ac_compress_dir
 *   trim_path_start_end / _hairpin_start / _hairpin_end   trim.rs:288-326 -> ac_trim_paths
 *   trim.rs:43-51 on a loaded graph (trim minus the file I/O)     -> ac_trim
 *   trim (the whole subcommand)             trim.rs:36-53            -> ac_trim_dir, ac_trim_dirs (several clusters)
 *   Bridge::new (best path of a bridge)     resolve.rs:430-462       -> ac_bridge_best_paths
 *   resolve.rs:41-67 on a loaded graph                               -> ac_resolve, ac_resolve_text, ac_resolve_stats
 *   resolve / combine (the whole subcommands)  resolve.rs:31-69, combine.rs:25-49 -> ac_resolve_dir, ac_resolve_dirs, ac_combine_dir
 *   clean (the whole subcommand)            clean.rs:23-149          -> ac_clean_gfa
 *   clean.rs:26-45 on a GFA text            unitig_graph.rs:588-721  -> ac_clean_text
 *   gfa2fasta (the whole subcommand)        gfa2fasta.rs:23-82       -> ac_gfa_to_fasta, ac_gfa_fasta_text
 *   table (the whole subcommand)            table.rs:24-204, misc.rs:373-386 -> ac_table_text
 *   create_dotplot without the file         dotplot.rs:179-221       -> ac_dotplot_rgb
 *   dotplot (the whole subcommand)          dotplot.rs:44-52         -> ac_dotplot_dir, ac_png_write
 *   subsample (the whole subcommand)        subsample.rs:29-43       -> ac_subsample_dir
 *   parse_genome_size                       subsample.rs:83-101      -> ac_genome_size
 *   StdRng::seed_from_u64 + shuffle         subsample.rs:151-153     -> ac_subsample_words, ac_subsample_shuffle
 *   helper genome_size                      helper.rs:388-403        -> ac_genome_size_estimate, ac_genome_size_from_histogram
 *       (a deliberate departure: a k-mer depth estimate from the reads on the GPU, not the length of a Raven assembly)
 *   depth_filter, depth_from_header         helper.rs:889-931        -> ac_depth_filter_text, ac_depth_from_header
 *   depth (read-measured contig depth)      not in the reference     -> ac_depth_fasta
 *   qv (k-mer QV and completeness)          not in the reference     -> ac_qv_dir
 *   unassembled (reads the assembly lacks)  not in the reference     -> ac_unassembled_dir
 *   polish (k-mer consensus correction)     not in the reference     -> ac_polish_fasta
 *   variants (alleles beside the consensus) not in the reference     -> ac_variants_fasta
 *
 * Conventions: every function returns 0 on success and a negative AC_E* code on failure; the message
 * is available from ac_last_error(handle) (or ac_last_error(NULL) when no handle exists).  No C++
 * exception crosses the boundary.  The caller owns every buffer it passes; inputs are copied during
 * the call; outputs are written into caller-allocated buffers sized from ac_counts_get / ac_gfa_size.
 * A handle must be used from one host thread at a time (the reference path is single-threaded and
 * !Send).  There is no CPU fallback: without a CUDA device ac_create fails with AC_ENODEVICE.
 */
#ifndef AUTOCYCLER_GPU_H
#define AUTOCYCLER_GPU_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AC_OK 0
#define AC_EINVAL (-1)      /* bad argument (even k, k out of range, non-ACGT. byte, call order) */
#define AC_ENODEVICE (-2)   /* no usable CUDA device */
#define AC_ECUDA (-3)       /* CUDA runtime error */
#define AC_ERANGE (-4)      /* buffer too small / input too large */
#define AC_EIO (-5)         /* file system error: an input that cannot be read, an output that cannot be written (the commands) */
#define AC_EINPUT (-6)      /* the reference's own input errors (misc.rs:130-136 quit_with_error) */

typedef struct ac_handle ac_handle;

typedef struct {
    uint32_t k;             /* odd; 3..511 (compress.rs:56-58 restricts the CLI to 11..501) */
    int32_t device;         /* CUDA device ordinal */
    void* stream;           /* cudaStream_t to run on, or NULL for a private (non-blocking) stream; the default stream is named by its handle (cudaStreamLegacy / cudaStreamPerThread) */
    uint32_t keep_positions;/* non-zero: ac_unitigs_copy can return full forward/reverse position lists */
    int32_t n_devices;      /* > 1: this ONE process drives several GPUs (SURVEY.md 8b/8e): the assemblies are sharded by file over */
    const int32_t* devices; /* devices[0..n_devices) (devices[0] finishes the graph; `device` and `stream` are ignored); 0/1: one GPU, `device` */
} ac_config;

typedef struct {
    uint64_t n_kmers;       /* both strands == KmerGraph.kmers.len() printed at compress.rs:152 */
    uint64_t n_unitigs;
    uint64_t n_links;       /* UnitigGraph::link_count().1 (unitig_graph.rs:478-507) */
    uint64_t total_length;  /* UnitigGraph::total_length (unitig_graph.rs:474-476) */
    uint64_t seq_bytes;     /* sum of unitig sequence lengths for ac_unitigs_copy (trimmed) */
    uint64_t n_fwd_pos, n_rev_pos;   /* total entries of forward_positions / reverse_positions */
    uint64_t n_next;        /* total entries of forward_next + reverse_next */
    uint64_t n_sequences;
    uint64_t n_path_steps;  /* sum of path lengths over all sequences */
    uint64_t length_before_simplify;   /* total_length() of the graph as built, before simplify_structure moved bases (compress.rs:164) */
} ac_counts;

/* Unitigs in the graph's current order (after ac_build: the order renumber_unitigs gives, numbers 1..U).
 * All arrays are caller-allocated from ac_counts; offsets arrays have n_unitigs+1 entries. */
typedef struct {
    uint32_t* number;       /* [U] Unitig.number */
    uint64_t* seq_off;      /* [U+1] */
    uint8_t* seq;           /* [seq_bytes] forward_seq, ASCII */
    double* depth;          /* [U] Unitig.depth */
    uint64_t* fpos_off;     /* [U+1]; positions need ac_config.keep_positions, else pass NULL */
    uint32_t* fpos;         /* [n_fwd_pos] Position.pos (position.rs:20) */
    uint16_t* fpos_id_strand; /* [n_fwd_pos] Position.seq_id_and_strand (position.rs:21; bit 15 = forward strand) */
    uint64_t* rpos_off; uint32_t* rpos; uint16_t* rpos_id_strand;
    uint64_t* next_off;     /* [2U+1] forward_next of unitig i at 2i, reverse_next at 2i+1 */
    int32_t* next;          /* [n_next] signed unitig numbers, negative = reverse strand (UnitigStrand::signed_number) */
} ac_unitigs;

typedef struct {            /* milliseconds */
    float h2d, pack, insert, adjacency, boundaries, runs, unitigs, links, seed_sort, emit, d2h, device_total;
    float host_graph, host_simplify, host_gfa;
    float sample, device_simplify, device_gfa;   /* sizing pass of the k-mer table; expand_repeats passes + renumbering and the GFA text when they run on the device */
    float insert_kernel;                         /* the hash-insert kernel alone (CUDA events right around its launch; `insert` also holds the table initialisation and the counter read-back) */
    float trim_kernel;                           /* ac_trim / ac_trim_paths: the overlap-alignment kernels alone (CUDA events around their launches), summed over the call's rounds */
    uint64_t insert_occurrences;   /* k-mer occurrences hashed by the insert kernel (forward windows; each feeds both strands) */
    uint64_t table_capacity, table_used;
    uint64_t kernel_launches;      /* cumulative launches of this library's kernels in the process */
    uint64_t h2d_bytes, d2h_bytes; /* bytes moved by ac_upload / ac_build */
} ac_timings;

const char* ac_last_error(const ac_handle* h);
const char* ac_version(void);

int ac_create(ac_handle** out, const ac_config* cfg);
void ac_destroy(ac_handle* h);

/* One padded, end-repaired forward strand (Sequence.forward_seq after compress.rs:125, bytes in "ACGT.",
 * k/2 dots or repaired bases at both ends) with the fields save_gfa prints (unitig_graph.rs:352-360). */
int ac_add_sequence(ac_handle* h, uint16_t seq_id, const uint8_t* fwd_padded, uint64_t padded_len,
                    const char* filename, const char* contig_header);
int ac_clear_sequences(ac_handle* h);
int ac_upload(ac_handle* h);            /* host -> HBM copy of the added sequences */
/* Multi-GPU: copy only the strands of sequences [seq_lo, seq_hi) over this process's PCIe link; the other ranks' blocks are brought
 * over NVLink by the caller's collective, each into the device range ac_strand_block names for it (blocks tile the strand buffer). */
int ac_upload_shard(ac_handle* h, uint32_t seq_lo, uint32_t seq_hi);
int ac_strand_block(ac_handle* h, uint32_t seq_lo, uint32_t seq_hi, void** dev_ptr, uint64_t* n_bytes);
int ac_build(ac_handle* h);             /* k-mer table, unitigs, links, renumber: the graph after from_kmer_graph */
int ac_simplify(ac_handle* h);          /* simplify_structure */
/* compress.rs:42-47 in one call — build_kmer_graph, build_unitig_graph, simplify_unitig_graph and the bytes save_gfa writes — as ONE
 * device pipeline: repeat expansion, the closing renumbering and the H/S/L/P text are produced by kernels and only the text and the
 * counts compress prints travel back.  Afterwards ac_gfa_* return the file, ac_counts_get the counts (length_before_simplify = the
 * graph as built); the graph arrays stay in HBM and are fetched the first time a call needs them (ac_unitigs_copy, ac_path_copy,
 * ac_merge_linear_paths, ...).  `autocycler compress`, ac_compress_dir and bench.py use this call. */
int ac_compress(ac_handle* h);
/* merge_linear_paths (graph_simplification.rs:315-371), what cluster/trim/resolve/clean first do to a loaded compress
 * graph (cluster.rs:804): chains of exclusively linked unitigs become one unitig numbered max+1, max+2, ...; merged
 * unitigs follow the surviving ones in the S lines.  use_paths != 0 keeps sequence-path ends fixed (the reference's
 * `seqs` argument); 0 is its `&vec![]` form: everything mergeable is merged and the P lines lose their paths. */
int ac_merge_linear_paths(ac_handle* h, int use_paths);
/* renumber_unitigs (unitig_graph.rs:295-315) on the current graph, e.g. after ac_merge_linear_paths as trim.rs:266-268 does. */
int ac_renumber_unitigs(ac_handle* h);

/* Multi-GPU form of ac_build (SURVEY.md 8e): one process per GPU, every process adds and uploads ALL sequences, owns the
 * contiguous block [seq_lo, seq_hi) of them (index = order of ac_add_sequence), and the caller (e.g. torch.distributed over
 * NCCL) moves the exported records between the processes.  Buffers are device memory on the handle's device.
 *   ac_build_local -> ac_entries_count/export -> [all-gather] -> ac_entries_merge (every other rank's records)
 *   -> ac_runs_local -> ac_runs_export -> [gather to rank 0] -> rank 0: ac_runs_import (all ranks, rank order) -> ac_build_finish
 * Records are opaque: 16 bytes per k-mer entry, 16 bytes per unitig occurrence.  ac_runs_import_padded reads the buffer a padded
 * gather leaves behind (rank r's counts[r] records start at record r * stride_records); ac_compress_finish is ac_compress for the
 * importing rank (simplify_structure and the GFA text on the device as well).
 * The buffers passed to ac_entries_merge must stay valid, unchanged, until ac_runs_local returns: when the other ranks' k-mers overflow
 * a table sized from the estimate, ac_runs_local builds this rank's table again at the safe size and folds the same records in again. */
int ac_build_local(ac_handle* h, uint32_t seq_lo, uint32_t seq_hi, uint32_t multi);
int ac_entries_count(ac_handle* h, uint64_t* n);
int ac_entries_export(ac_handle* h, void* dst, uint64_t cap_records);
int ac_entries_merge(ac_handle* h, const void* src, uint64_t n);
int ac_runs_local(ac_handle* h, uint64_t* n_runs);
int ac_runs_export(ac_handle* h, void* dst, uint64_t cap_records);
int ac_runs_import(ac_handle* h, const void* src, uint64_t n);
int ac_runs_import_padded(ac_handle* h, const void* src, uint64_t stride_records, const uint64_t* counts, uint32_t n_ranks);
int ac_build_finish(ac_handle* h);      /* on the rank that imported the runs: the graph after from_kmer_graph */
int ac_compress_finish(ac_handle* h);
/* The same with the P lines printed where the sequences live (the GFA of many assemblies is mostly P lines; one rank printing and
 * copying out all of them is what bounds the scaling):
 *   rank 0 (it must own the first block of sequences): ac_compress_finish_split — ac_gfa_data then ends after the L lines —
 *   -> ac_path_tokens_export: one uint32 per occurrence, "(final unitig number - 1) << 1 | strand", rank r's counts[r] tokens at
 *   dst + r * stride_tokens (the counts given to ac_runs_import_padded) -> [scatter] -> every rank: ac_path_lines_render with the tokens
 *   of its own occurrences -> ac_path_lines_data: the P lines of its own sequences (unitig_graph.rs:352-360), pinned host memory.
 * input_assemblies.gfa = rank 0's text followed by the ranks' path lines in rank order. */
int ac_compress_finish_split(ac_handle* h);
int ac_path_tokens_export(ac_handle* h, void* dst, uint64_t stride_tokens, const uint64_t* counts, uint32_t n_ranks);
int ac_path_lines_render(ac_handle* h, const void* tokens, uint64_t n_tokens);
int ac_path_lines_data(ac_handle* h, const char** data, uint64_t* n_bytes);   /* borrowed: valid until the next call on h */
int ac_counts_get(const ac_handle* h, ac_counts* out);
int ac_unitigs_copy(const ac_handle* h, ac_unitigs* out);
int ac_path_copy(const ac_handle* h, uint64_t seq_index, int32_t* out, uint64_t cap, uint64_t* n);  /* get_unitig_path_for_sequence_i32 */
int ac_gfa_size(ac_handle* h, uint64_t* n_bytes);
int ac_gfa_copy(ac_handle* h, char* buf, uint64_t cap);
int ac_gfa_data(ac_handle* h, const char** data, uint64_t* n_bytes);   /* the same bytes, borrowed: valid until the next call on h */
int ac_timings_get(const ac_handle* h, ac_timings* out);

/* `autocycler compress -i assemblies_dir -a autocycler_dir --kmer k --max_contigs m -t threads`
 * (main.rs:126-147, compress.rs:32-50): writes input_assemblies.gfa and input_assemblies.yaml.
 * ac_compress_dir_devices is the same on several GPUs of one box (`autocycler compress --devices 0,1,...`): the assemblies are
 * sharded by file, one contiguous block of files per device, the k-mer buckets are read across NVLink by the peers' merge kernels. */
int ac_compress_dir(const char* assemblies_dir, const char* autocycler_dir, uint32_t k, uint32_t max_contigs,
                    uint32_t threads, int32_t device, int32_t verbose);
int ac_compress_dir_devices(const char* assemblies_dir, const char* autocycler_dir, uint32_t k, uint32_t max_contigs,
                            uint32_t threads, const int32_t* devices, int32_t n_devices, int32_t verbose);

/* Host-side stage A of compress (compress.rs:98-133): directory scan, FASTA load, padding, end repair.
 * Fills a handle created with the same k, ready for ac_upload.  Returns the number of assemblies. */
int ac_load_sequences(ac_handle* h, const char* assemblies_dir, uint32_t max_contigs, uint32_t threads,
                      uint64_t* assembly_count);
/* Read back one loaded sequence (for tests of stage A): padded forward strand and header fields. */
int ac_sequence_get(const ac_handle* h, uint64_t index, uint16_t* seq_id, uint64_t* length,
                    char* fwd_padded, uint64_t cap_fwd, char* filename, uint64_t cap_fn, char* header, uint64_t cap_hd);

/* UnitigGraph::from_gfa_lines (unitig_graph.rs:55-174): replaces whatever the handle holds by the graph and the sequences of an
 * Autocycler GFA (H/S/L/P lines; `length` bytes of text), so that the calls above that work on a built graph — ac_gfa_*,
 * ac_sequence_reconstruct (decompress.rs:83-105), ac_merge_linear_paths, ac_simplify, ac_renumber_unitigs, ac_counts_get,
 * ac_unitigs_copy, ac_path_copy — apply to a file written earlier.  Host only.  Any DP:f: value the reference parses (f64) and the
 * CL:Z: segment colours (UnitigType, unitig.rs:72-86) are carried and written back; lines may end in "\r\n" (misc.rs:51-61).
 * Errors: the reference's own (missing tags, unknown unitigs, non-zero overlaps ...). */
int ac_load_gfa(ac_handle* h, const char* gfa_text, uint64_t length);

/* Deployment helper, not part of the reference: restricts the calling thread (and the threads created after it) to the CPUs of the
 * NUMA node the CUDA device is attached to, so that pinned host buffers are local to both.  Returns the node (>= 0) or a negative
 * AC_E* with the affinity unchanged.  Call it before ac_create; `autocycler compress` and bench.py do. */
int ac_bind_host_to_device(int32_t device);

/* pairwise_contig_distances (cluster.rs:132-151), the all-against-all step of `autocycler cluster`: out[a * S + b] for the S sequences of
 * the handle (built or loaded graph); the unitig-set intersections are computed on the GPU.  ac_distance_matrix_text renders
 * save_distance_matrix's file (cluster.rs:160-176); `out` may be NULL to query the length. */
int ac_pairwise_distances(ac_handle* h, double* out, uint64_t cap);
int ac_distance_matrix_text(ac_handle* h, char* out, uint64_t cap, uint64_t* length);

/* `autocycler decompress` (decompress.rs:27-137): every contig of the GFA's paths written back per original file under out_dir
 * (gzip when the name ends in .gz) and/or as one FASTA (out_file); either may be NULL, not both.  A malformed GFA is AC_EINPUT. */
int ac_decompress_gfa(const char* in_gfa, const char* out_dir, const char* out_file, int32_t device, int32_t verbose);

/* reconstruct_original_sequence (unitig_graph.rs:383-400; decompress.rs:83-105 writes these out): the sequence spelled by
 * the path of loaded/added sequence `index` through the current graph.  `out` may be null to query `length` only. */
int ac_sequence_reconstruct(const ac_handle* h, uint64_t index, char* out, uint64_t cap, uint64_t* length);

/* `autocycler trim`.  The overlap alignments (trim.rs:366-479: a dense (k+1)^2 f64 DP per alignment, k = min(max_unitigs, path
 * length)) run on the GPU, one CTA per alignment, with the traceback on the device; the identity test, the midpoint and the hairpin
 * walk run on the host.  There is no CPU path: the emulation build exists for the test-suite only. */
#define AC_TRIM_START_END 0       /* trim_path_start_end (trim.rs:288-296) */
#define AC_TRIM_HAIRPIN_START 1   /* trim_path_hairpin_start (trim.rs:320-326) */
#define AC_TRIM_HAIRPIN_END 2     /* trim_path_hairpin_end (trim.rs:299-317) */
/* One `mode` trim for each of n_paths paths: path x is paths[path_off[x] .. path_off[x+1]) (signed unitig numbers, negative = reverse
 * strand); weights[u] = length of unitig u (n_weights entries, every |unitig| below n_weights).  trimmed[x] = 1 when path x was
 * trimmed, and then out[out_off[x] .. out_off[x+1]) is the trimmed path; otherwise that range is empty.  out needs room for
 * path_off[n_paths] values (a trimmed path is never longer than its input).  The reference's trim.rs unit tests run through this call. */
int ac_trim_paths(ac_handle* h, int32_t mode, const int32_t* paths, const uint64_t* path_off, uint64_t n_paths,
                  const uint32_t* weights, uint64_t n_weights, double min_identity, uint32_t max_unitigs,
                  int32_t* out, uint64_t* out_off, uint8_t* trimmed);
/* trim.rs:43-51 on the handle's graph (ac_load_gfa of a 1_untrimmed.gfa): start-end and hairpin trimming, choose_trim_type, length
 * outliers (mad = 0 disables), clean-up (recalculate_depths, remove_zero_depth_unitigs, merge_linear_paths, renumber_unitigs).
 * Afterwards ac_gfa_*, ac_counts_get, ac_path_copy and ac_sequence_get describe 2_trimmed.gfa and its sequences, ac_trim_yaml returns
 * 2_trimmed.yaml (TrimmedClusterMetrics, metrics.rs:209-225) and ac_timings.trim_kernel the alignment kernels' time. */
int ac_trim(ac_handle* h, double min_identity, uint32_t max_unitigs, double mad);
int ac_trim_yaml(ac_handle* h, char* out, uint64_t cap, uint64_t* length);   /* `out` may be NULL to query the length */
/* What the last ac_trim / ac_trim_paths aligned: alignments, DP cells (sum of k^2), the largest window k and the longest path. */
int ac_trim_stats(const ac_handle* h, uint64_t* jobs, uint64_t* cells, uint32_t* max_window, uint64_t* max_path);
/* `autocycler trim -c cluster_dir` (main.rs:302-322, trim.rs:36-67): reads 1_untrimmed.gfa, writes 2_trimmed.gfa and 2_trimmed.yaml.
 * The reference's setting checks and messages (AC_EINPUT). */
int ac_trim_dir(const char* cluster_dir, double min_identity, uint32_t max_unitigs, double mad, uint32_t threads, int32_t device, int32_t verbose);

/* Several clusters in one call (ac_trim_dirs, ac_resolve_dirs): every cluster goes through each phase, and each device step is one
 * call over all of them, so a trim makes at most four kernel launches and a resolve at most two, whatever the number of clusters.
 * Every directory's outputs are byte for byte those of the single-directory call.  Every directory is checked, read and loaded before
 * any device work, and files are written only after every cluster has finished: an error writes nothing, and it is the error the
 * single-directory call gives for the first failing directory in argument order.  A directory given twice (after realpath) is
 * AC_EINPUT "cluster directory given twice: <dir>"; a rebased unitig number at or above 2^31 is AC_ERANGE.
 * verbose: AC_VERBOSE_REPORT for the single call's report and AC_VERBOSE_BANNER for the `Starting autocycler <command> (<version>)`
 * block the command-line tool prints, per directory, in argument order, after the last cluster finishes.  With more than one directory
 * the reports leave out the kernel time, which a shared launch cannot split by cluster, and one closing line gives the batch's totals. */
#define AC_VERBOSE_REPORT 1
#define AC_VERBOSE_BANNER 2
typedef struct {
    uint32_t clusters;                 /* directories */
    uint32_t launches;                 /* kernel launches made */
    uint64_t jobs;                     /* alignments (trim) or distance jobs (resolve) */
    uint64_t cells;                    /* DP cells: sum of k^2 (trim) or n * m (resolve) */
    uint64_t buffer_bytes;             /* the largest device call's planned buffers: jobs, paths, weights, scratch and outputs */
    float kernel_ms;                   /* CUDA events around the launches; 0 under emulation */
} ac_batch_info;
/* `autocycler trim -c dir [dir ...]`: ac_trim_dir for n cluster directories with the same settings.  info may be NULL. */
int ac_trim_dirs(const char* const* cluster_dirs, uint32_t n, double min_identity, uint32_t max_unitigs, double mad, uint32_t threads,
                 int32_t device, int32_t verbose, ac_batch_info* info);

/* `autocycler cluster`.  The contig distances (cluster.rs:132-192) and UPGMA (:395-480) run on the GPU: the symmetric matrix stays in
 * HBM and one persistent CTA performs all n - 1 merges; the tree, clustering, QC and the output files are built on the host.  Averages
 * are kept as sums over member pairs (T(A u B, C) = T(A, C) + T(B, C)), see DESIGN.md section 12. */
#define AC_CLUSTER_PHYLIP 0            /* pairwise_distances.phylip */
#define AC_CLUSTER_NEWICK 1            /* clustering.newick */
#define AC_CLUSTER_TSV 2               /* clustering.tsv */
#define AC_CLUSTER_YAML 3              /* clustering.yaml (ClusteringMetrics) */
#define AC_CLUSTER_GFA 4               /* one cluster's 1_untrimmed.gfa */
#define AC_CLUSTER_UNTRIMMED_YAML 5    /* one cluster's 1_untrimmed.yaml (UntrimmedClusterMetrics) */
/* cluster.rs:42-59 on the handle's graph as it is now (normally ac_load_gfa of an input_assemblies.gfa): the distances and the
 * per-cluster graphs both come from it.  The handle's sequences and graph are not changed.  min_assemblies < 0: set automatically;
 * manual: n_manual node numbers of the tree (none: automatic clustering refined by score).  The reference's setting checks (AC_EINPUT);
 * two sequences whose paths have no length have a NaN distance and are refused (AC_EINPUT), where the reference would panic. */
int ac_cluster(ac_handle* h, double cutoff, int64_t min_assemblies, const uint16_t* manual, uint64_t n_manual);
/* One output of the last ac_cluster (`what` = AC_CLUSTER_*; `cluster` = 1-based number for the per-cluster texts).  `out` may be NULL
 * to query the length. */
int ac_cluster_text(ac_handle* h, int32_t what, uint32_t cluster, char* out, uint64_t cap, uint64_t* length);
/* Per sequence of the handle: its cluster number and whether that cluster passed QC. */
int ac_cluster_assignments(const ac_handle* h, uint16_t* cluster, uint8_t* pass, uint64_t cap);
/* The last ac_cluster: sequences, passed and failed clusters, the distance and UPGMA kernels' times (CUDA events) and the host time of
 * the per-cluster graphs. */
int ac_cluster_stats(const ac_handle* h, uint32_t* n_seqs, uint32_t* pass_clusters, uint32_t* fail_clusters, float* distance_ms, float* upgma_ms,
                     double* cluster_gfa_ms);
/* The UPGMA kernel on a caller's symmetric n x n matrix (row-major) of the clusters ids[0..n), strictly ascending: n - 1 merges, each
 * the new node's number (from ids[n-1] + 1), its left and right child and its distance to the tips.  A NaN off the diagonal is refused
 * (AC_EINPUT).  The reference's UPGMA tests run through this call. */
int ac_upgma(ac_handle* h, const double* sym_dist, uint32_t n, const uint32_t* ids, uint32_t* node, uint32_t* left, uint32_t* right, double* dist);
/* `autocycler cluster -a autocycler_dir` (main.rs:92-113, cluster.rs:30-64): replaces autocycler_dir/clustering with
 * pairwise_distances.phylip, clustering.newick, clustering.tsv, clustering.yaml and qc_pass|qc_fail/cluster_NNN/1_untrimmed.{gfa,yaml}.
 * min_assemblies < 0: automatic; manual: "1,2,3" or NULL. */
int ac_cluster_dir(const char* autocycler_dir, double cutoff, int64_t min_assemblies, uint32_t max_contigs, const char* manual, int32_t device, int32_t verbose);

/* `autocycler resolve` and `autocycler combine`.  The one step of resolve whose cost grows quadratically — global_alignment_distance
 * (resolve.rs:387-418) between every pair of a bridge's paths (Bridge::new, :430-462) — runs on the GPU: identical paths are aligned
 * once, each pair of distinct paths is one CTA sweeping the anti-diagonals of a u32 DP (shared memory, or HBM scratch for paths beyond
 * it), all bridges in one launch per storage form.  Anchors, bridges, ambiguity, culling and the graph edits run on the host
 * (DESIGN.md section 13).  combine needs no device. */
#define AC_RESOLVE_BRIDGED 0           /* 3_bridged.gfa */
#define AC_RESOLVE_MERGED 1            /* 4_merged.gfa */
#define AC_RESOLVE_FINAL 2             /* 5_final.gfa */
typedef struct {
    uint32_t anchors;                  /* anchor unitigs */
    uint32_t unique_bridges, conflicting_bridges, culled_bridges;
    uint64_t jobs;                     /* distance jobs: pairs of distinct trimmed paths of one bridge */
    uint64_t cells;                    /* sum of n * m over the jobs */
    uint64_t longest_path;             /* longest trimmed bridge path (unitigs) */
    uint32_t shared_jobs, hbm_jobs;    /* jobs whose three diagonals sat in shared memory / in HBM scratch */
    float kernel_ms;                   /* the distance kernels alone (CUDA events around their launches; 0 under emulation) */
} ac_resolve_info;
/* Bridge::new for n_groups bridges at once: group g holds paths group_off[g] .. group_off[g+1] (indices into the path list), path x is
 * paths[path_off[x] .. path_off[x+1]) (signed unitig numbers: a bridge's paths with the start and end anchors already removed);
 * weights[u] = length of unitig u (every |unitig| below n_weights).  totals[x] = path x's u32 (wrapping) sum of distances to the other
 * paths of its group; best[best_off[g] .. best_off[g+1]) = the path the reference selects for group g (least total, ties to the
 * lexicographically smaller path; empty when every total is u32::MAX).  best needs room for path_off[n_paths] values.  The reference's
 * resolve.rs unit tests run through this call. */
int ac_bridge_best_paths(ac_handle* h, const int32_t* paths, const uint64_t* path_off, uint64_t n_paths, const uint64_t* group_off, uint64_t n_groups,
                         const uint32_t* weights, uint64_t n_weights, uint32_t* totals, int32_t* best, uint64_t* best_off);
/* resolve.rs:41-67 on the handle's graph (ac_load_gfa of a 2_trimmed.gfa): anchors, bridges, the unique bridges applied, culling and,
 * when anything was culled, the final bridges applied to the graph as loaded.  The handle's graph is not changed; the three files are
 * available from ac_resolve_text, the counts and the kernel time from ac_resolve_stats.  verbose: a report on stderr. */
int ac_resolve(ac_handle* h, int32_t verbose);
int ac_resolve_text(ac_handle* h, int32_t what, char* out, uint64_t cap, uint64_t* length);   /* `out` may be NULL to query the length */
int ac_resolve_stats(const ac_handle* h, ac_resolve_info* out);
/* `autocycler resolve -c cluster_dir` (main.rs:238-247, resolve.rs:31-75): reads 2_trimmed.gfa, writes 3_bridged.gfa, 4_merged.gfa and
 * 5_final.gfa.  The reference's checks (AC_EINPUT). */
int ac_resolve_dir(const char* cluster_dir, int32_t verbose, int32_t device);
/* `autocycler resolve -c dir [dir ...]`: ac_resolve_dir for n cluster directories, as ac_trim_dirs does for trim.  info may be NULL. */
int ac_resolve_dirs(const char* const* cluster_dirs, uint32_t n, int32_t verbose, int32_t device, ac_batch_info* info);
/* `autocycler combine -a autocycler_dir -i gfa [gfa ...]` (main.rs:115-124, combine.rs:25-137): writes consensus_assembly.gfa, .fasta and
 * .yaml under autocycler_dir (created if needed) from the n_gfas GFAs in argument order.  Host only. */
int ac_combine_dir(const char* autocycler_dir, const char* const* in_gfas, uint32_t n_gfas, int32_t verbose);

/* `autocycler clean`, `autocycler gfa2fasta` and `autocycler table`: host only, no device and no handle.  The getters follow the
 * two-call convention: `out` NULL asks for the length, then a buffer of that size takes the text (AC_ERANGE when `cap` is short).
 * The reference's input errors are AC_EINPUT, with its messages; a tig both removed and duplicated, and a tig duplicated twice, which
 * make the reference panic, are AC_EINPUT too.
 *
 * `autocycler clean -i in_gfa -o out_gfa [-r LIST] [-d LIST] [-m DEPTH]` (main.rs:69-90, clean.rs:23-149): remove and duplicate are the
 * comma-separated tig lists (NULL for none), min_depth is NULL for none.  Removes, duplicates, drops low-depth tigs that leave no dead
 * end, merges linear paths, renumbers and saves (Other unitigs CL:Z:orangered, no P lines). */
int ac_clean_gfa(const char* in_gfa, const char* out_gfa, const char* remove, const char* duplicate, const double* min_depth, int32_t verbose);
/* clean.rs:26-45 on a GFA text with the tig numbers already parsed (any order).  merge = 0 stops before merge_linear_paths and
 * renumber_unitigs and saves the edited graph in its list order. */
int ac_clean_text(const char* gfa_text, uint64_t length, const uint32_t* remove, uint64_t n_remove, const uint32_t* duplicate,
                  uint64_t n_duplicate, const double* min_depth, int32_t merge, char* out, uint64_t cap, uint64_t* out_length);
/* `autocycler gfa2fasta -i in_gfa -o out_fasta` (main.rs:183-192, gfa2fasta.rs:23-82): every non-empty unitig in the file's order,
 * with circular=true / circular=false topology in the headers. */
int ac_gfa_to_fasta(const char* in_gfa, const char* out_fasta, int32_t verbose);
int ac_gfa_fasta_text(const char* gfa_text, uint64_t length, char* out, uint64_t cap, uint64_t* out_length);   /* save_graph_to_fasta's text */
/* `autocycler table [-a dir] [-n name] [-f fields] [-s sigfigs]` (main.rs:276-299, table.rs:24-204): with autocycler_dir NULL the header
 * line, else the name and each field's value from the directory's YAML files, tab-separated, newline included.  fields NULL takes the
 * reference's default list.  verbose: the "not found" warnings on stderr.  Unlike the reference, nothing is printed before an error. */
int ac_table_text(const char* autocycler_dir, const char* name, const char* fields, uint64_t sigfigs, int32_t verbose, char* out, uint64_t cap,
                  uint64_t* length);

/* `autocycler dotplot`.  The all-vs-all k-mer dots (dotplot.rs:202-211, 394-450) run on the GPU: every window of only ACGT gets its
 * canonical k-mer, the windows are grouped by it, and each ordered pair of windows in a group is one dot whose 64-bit key (pair of
 * sequences, window, forward) goes into a per-pixel maximum, which fixes the colour the reference's loop order leaves.  Windows with
 * other bytes are matched on the host by the reference's literal rules and merged into the same maxima.  The layout, the boxes, the
 * labels (a TrueType font read at run time) and the PNG are host work (DESIGN.md section 14).
 *
 * font: a TrueType file for the labels; "" draws no labels; NULL takes the first of a fixed list of standard DejaVuSans.ttf paths that
 * exists (none: no labels, and ac_dotplot_dir prints one warning line).  Without labels the layout is the one the reference uses when
 * its labels fit at the largest font size.
 *
 * Calls on one device run one at a time (a lock around the device work).  The device buffers of a call stay allocated for the next
 * call on that device until the process ends: about 70 to 80 bytes per window and 8 bytes per pixel (res * res). */
typedef struct {
    uint64_t windows;                  /* k-mer windows over every sequence (len - k + 1 each) */
    uint64_t groups;                   /* distinct canonical k-mers among the windows of only ACGT */
    uint64_t dots;                     /* dots, including those that fall outside the image: the groups' squared sizes plus the host's */
    uint64_t host_windows;             /* windows holding a byte other than ACGT, matched on the host */
    double bp_per_pixel;               /* get_positions (dotplot.rs:268-269) */
    float text_height;                 /* reduce_scale's font size (dotplot.rs:308-327) */
    float kernel_ms;                   /* CUDA events from the first to the last dot kernel (0 under emulation); the span includes two
                                          blocking reads of a count by the host (the group count and the dot count) */
} ac_dotplot_info;
/* create_dotplot (dotplot.rs:179-221) for n sequences: seqs[i] holds lengths[i] bytes (uppercased here; bytes other than ACGT are kept),
 * labelled (filenames[i] or "" when filenames is NULL, names[i]); no two labels may be equal (AC_EINPUT).  rgb: res * res * 3 bytes,
 * row-major RGB.  The reference's --res and --kmer checks apply (AC_EINPUT).  info may be NULL. */
int ac_dotplot_rgb(const char* const* seqs, const uint64_t* lengths, const char* const* filenames, const char* const* names, uint32_t n,
                   uint32_t res, uint32_t kmer, const char* font, int32_t device, uint8_t* rgb, ac_dotplot_info* info);
/* `autocycler dotplot -i input -o out_png --res R --kmer K [--font F]` (main.rs:164-181, dotplot.rs:44-52): input is a directory of
 * assemblies, a FASTA file or an Autocycler GFA (gzipped or not).  The reference's checks and messages (AC_EINPUT).  info may be NULL. */
int ac_dotplot_dir(const char* input, const char* out_png, uint32_t res, uint32_t kmer, const char* font, int32_t device, int32_t verbose,
                   ac_dotplot_info* info);
/* rgb (width * height * 3 bytes, row-major) as an 8-bit RGB PNG at path.  Host only. */
int ac_png_write(const char* path, const uint8_t* rgb, uint32_t width, uint32_t height);

/* `autocycler subsample -r reads -o out_dir -g genome_size [-c count] [-d min_read_depth] [-s seed]` (main.rs:249-274,
 * subsample.rs:29-43).  The FASTQ file (gzipped or not; every gzip member is read) streams through windows of host and device memory;
 * the record scan, the read statistics (count, bases, the reference's ascending n50) and the split into subsets run on the GPU, the
 * seeded shuffle (rand 0.9's StdRng, ChaCha12) on the host.  Writes sample_01.fastq .. sample_NN.fastq and subsample.yaml as the
 * reference does (DESIGN.md section 16).  The reference's settings checks and messages in its order (AC_EINPUT); a malformed record is
 * AC_EINPUT "Error reading FASTQ file: record N: <reason>" before any sample file exists; 2^32 - 1 reads or more, or a read of 2^32
 * bases or more, is AC_ERANGE.  The window is 1 GiB unless AC_SUBSAMPLE_WINDOW gives another size in bytes; it grows for a record
 * longer than it.  When the file fits one window the second pass reuses the device copy, else the file is read again.
 * Calls on one device run one at a time.  info may be NULL. */
typedef struct {
    uint64_t genome_size;              /* parse_genome_size */
    uint64_t reads_per_subset;         /* calculate_subsets */
    uint64_t input_count, input_bases, input_n50;
    uint64_t windows;                  /* windows of the first pass */
    uint64_t bytes_scanned;            /* FASTQ bytes of the first pass (after gunzip) */
    float kernel_ms;                   /* CUDA events around each call's kernels, summed (0 under emulation); the spans include the host's
                                          reads of a count or an offset */
    double read_ms;                    /* host: reading and gunzipping the file, both passes */
    double shuffle_ms;                 /* host: the seeded shuffle */
    double write_ms;                   /* host: writing the sample files and subsample.yaml */
    double copy_ms;                    /* host wall time of the window uploads and the sample bytes' copies back */
} ac_subsample_info;
int ac_subsample_dir(const char* reads, const char* out_dir, const char* genome_size, uint64_t count, double min_read_depth, uint64_t seed,
                     int32_t device, int32_t verbose, ac_subsample_info* info);
/* parse_genome_size (subsample.rs:83-101): AC_EINPUT "cannot interpret genome size".  Host only. */
int ac_genome_size(const char* text, uint64_t* size);
/* The first n u32 words of StdRng::seed_from_u64(seed) (rounds 12), or of the same generator with 20 rounds (ChaCha20).  Host only. */
int ac_subsample_words(uint64_t seed, uint32_t rounds, uint32_t* out, uint64_t n);
/* (0..n).shuffle(&mut StdRng::seed_from_u64(seed)) (subsample.rs:151-153): order[p] = the read at shuffled position p.  Host only. */
int ac_subsample_shuffle(uint64_t n, uint64_t seed, uint32_t* order);

/* `autocycler helper genome_size -r reads [--kmer 21] [-d dir]`: the genome size from the reads' canonical k-mer depth spectrum.  This
 * departs from the reference on purpose: helper.rs:388-403 assembles the reads with Raven and reports the assembly's total length, which
 * this build cannot do, so the number differs from the reference's.  A replicon present in c copies per genome counts c times, and so
 * does each copy of a repeat (Raven's assembly holds one copy of each).  The FASTQ file streams through subsample's windows and record
 * scan (the same messages for a malformed record); every window is packed on the GPU at 2 bits and a validity bit per base; the canonical
 * k-mers are counted in partitions of an open-addressing table on the GPU and their counts binned into AC_GENOME_SIZE_BINS bins
 * (hist[c] = k-mers seen c times, the last bin every count at or above it).  The rule (DESIGN.md section 18): the valley v, the peak p,
 * the parabola vertex p*, and G = round((windows - sum_{c<v} c hist[c]) / p*).  k: odd, 11..31, else AC_EINPUT.  No k-mer windows:
 * AC_EINPUT; no depth peak: AC_EINPUT "no k-mer depth peak: ..."; a peak at the cap: AC_ERANGE.  dir (may be NULL): created if needed,
 * gets kmer_histogram.tsv (`count<TAB>k-mers` per non-zero bin).  hist (may be NULL): AC_GENOME_SIZE_BINS values.  The histogram file
 * and hist are written even when the rule then fails.  AC_GS_TABLE_SLOTS and AC_GS_PARTITIONS (DESIGN.md section 8) force a table
 * budget and a partition count.  Calls on one device run one at a time, with subsample's.  info may be NULL. */
#define AC_GENOME_SIZE_BINS 16384
typedef struct {
    uint64_t estimate;                 /* G, the genome size in bases */
    uint32_t k;
    uint32_t reruns;                   /* partitions counted again with twice the slots after their probe limit was hit */
    uint64_t reads, bases;             /* FASTQ records and their bases */
    uint64_t windows;                  /* W: windows of k A/C/G/T bases (any case) inside one read */
    uint64_t distinct;                 /* distinct canonical k-mers */
    uint64_t valley, peak;             /* v and p */
    double peak_refined;               /* p* */
    uint64_t solid;                    /* W - sum_{c<v} c hist[c], the numerator of G */
    uint64_t partitions;               /* P: passes over the packed stream, each with the table cleared */
    uint64_t table_bytes;              /* the largest table's bytes */
    float kernel_ms;                   /* CUDA events around every kernel, summed (0 under emulation) */
    float scan_ms, pack_ms, count_ms, hist_ms;   /* the same by stage: record scan, packing, counting, histogram */
    double read_ms;                    /* host: reading and gunzipping the file */
    double copy_ms;                    /* host wall time of the window uploads */
} ac_genome_size_info;
int ac_genome_size_estimate(const char* reads, uint32_t k, int32_t device, const char* dir, int32_t verbose, uint64_t* hist,
                            ac_genome_size_info* info);
/* The rule alone on a histogram of AC_GENOME_SIZE_BINS bins and its window count: info's estimate, windows, distinct, valley, peak,
 * peak_refined and solid (the rest 0).  AC_EINPUT for no depth peak or more occurrences below the valley than windows.  Host only. */
int ac_genome_size_from_histogram(const uint64_t* hist, uint64_t windows, ac_genome_size_info* info);

/* `autocycler depth -i assembly -o out.fasta [-r reads] [--source reads|header]`: each contig's read depth, and the reference's depth
 * filter (helper.rs:889-921).  Read-measured depth is an addition that is not in the reference (DESIGN.md section 19).
 * source_header = 0 (reads): reads is required (AC_EINPUT otherwise); the assembly is loaded as load_fasta does and a header that already
 * carries a depth (ac_depth_from_header) is AC_EINPUT.  Every contig window of k A/C/G/T bases (a contig whose header holds
 * "circular=true", any case, and whose length is at least k also gets the k-1 windows across its end) gives a canonical key; a key that
 * occurs once over all contigs is unique.  Each read window (the genome_size rule) whose key is a unique key adds 1 to it, on the GPU.
 * A contig's depth is the median of its unique keys' counts (the mean of the two middle ones for an even number); none without unique
 * keys.  out_fasta gets `>header[ depth={:.2}]\nseq\n` per contig; tsv (may be NULL) `name\tlength\tunique_kmers\tdepth` (empty without a
 * depth).  k: odd, 11..31, else AC_EINPUT.  A table beyond half the free device memory: AC_ERANGE.
 * source_header = 1: no reads are read and no device work runs: the assembly copied one line per sequence into out_fasta, as copy_fasta
 * does (nothing written, out_fasta removed, for a file without bases), then the filter.
 * The filter runs when min_abs or min_rel is given (may be NULL): nothing is filtered when a contig has no depth; otherwise the threshold
 * is max(min_abs or 0, min_rel x the depth of the first longest contig) and a contig is kept when its depth reaches it.  None kept: no
 * output file, and an existing one is removed.  verbose prints the settings, the depths and the filter's report to stderr.  depths and
 * unique (may be NULL) get the first `cap` contigs' depth (NaN: none) and unique keys (0 in header mode).  Calls on one device run one at
 * a time, with subsample's.  info may be NULL. */
typedef struct {
    uint64_t contigs;                  /* assembly records */
    uint64_t unique_kmers;             /* unique keys over all contigs */
    uint64_t assembly_windows;         /* the contigs' windows, junction windows included */
    uint64_t reads, read_windows, read_bases;
    uint64_t table_bytes;              /* the assembly table */
    uint64_t kept;                     /* records written to out_fasta */
    uint32_t k;
    int32_t filtered;                  /* 1 when the filter ran */
    float kernel_ms;                   /* CUDA events around every kernel, summed (0 under emulation) */
    float scan_ms, pack_ms, insert_ms, probe_ms, median_ms;   /* the same by stage: record scan, read packing, assembly table, probes, medians */
    double read_ms;                    /* host: reading and gunzipping the reads */
    double copy_ms;                    /* host wall time of the window uploads */
} ac_depth_info;
int ac_depth_fasta(const char* assembly, const char* reads, const char* out_fasta, const char* tsv, int32_t source_header, uint32_t k,
                   const double* min_abs, const double* min_rel, int32_t device, int32_t verbose, double* depths, uint64_t* unique,
                   uint64_t cap, ac_depth_info* info);
/* helper.rs:889-921 on a FASTA text: out gets what the file would hold afterwards: the text itself when the filter does not run (no bound
 * given, no bases, or a record without a depth), the kept records one line per sequence, or nothing when none is kept.  out NULL asks
 * for the length only.  Host only. */
int ac_depth_filter_text(const char* fasta_text, uint64_t length, const double* min_abs, const double* min_rel, char* out, uint64_t cap,
                         uint64_t* out_length);
/* helper.rs:923-931: the depth a header carries (depth=, then depth-, then coverage=).  AC_EINPUT when it carries none.  Host only. */
int ac_depth_from_header(const char* header, double* depth);

/* `autocycler qv -r reads -i assemblies... -o out_dir [--kmer 21] [--min_count N]`: each assembly's k-mer accuracy and completeness
 * against the reads (Merqury's QV and completeness), counted on the GPU.  Not in the reference (DESIGN.md section 20).  inputs: n_inputs
 * paths, each a FASTA file (gzipped or not, loaded as load_fasta does) or a directory, expanded as find_all_assemblies does.  Contig
 * windows are depth's (k A/C/G/T bases; a contig whose header holds "circular=true", any case, and whose length is at least k also gets the
 * k-1 windows across its end); read windows and the histogram are genome_size's.  r(key): the read windows with that canonical key.  The
 * solid threshold t is *min_count (1 .. AC_GENOME_SIZE_BINS - 1, else AC_EINPUT), or the histogram's valley when min_count is NULL (no
 * valley: AC_EINPUT "no k-mer depth peak: ...").  Per assembly: K windows, E of them with r < t, QV = -10 log10(-expm1(log1p(-E/K) / k))
 * (`%.2f`, "inf" for E = 0); S = the distinct read keys with count >= t; completeness = 100 x (its distinct keys with r >= t) / S.
 * out_dir (created if needed) gets qv.tsv, contig_qv.tsv, kmer_histogram.tsv (as helper genome_size -d writes it), unsupported/<n>.bed
 * (the merged stretches of bases covered by unsupported windows) and spectra_cn/<n>.tsv (Merqury's copy-number spectrum), n the
 * assembly's 1-based row.  k: odd, 11..31, else AC_EINPUT.  An assembly without windows, reads without windows: AC_EINPUT.  The tables
 * beyond half the free device memory: AC_ERANGE.  kmers, unsupported and solid_found (may be NULL) get the first `cap` assemblies' K, E
 * and found keys.  verbose prints the settings, the histogram's numbers and one line per assembly to stderr.  Calls on one device run one
 * at a time, with subsample's.  info may be NULL. */
typedef struct {
    uint64_t assemblies, contigs;
    uint32_t k;
    uint32_t min_count;                /* t, given or the valley */
    uint64_t valley;                   /* v of the reads' histogram (0: none) */
    uint64_t reads, read_windows, read_bases;
    uint64_t distinct;                 /* distinct canonical read k-mers */
    uint64_t solid_kmers;              /* S: distinct read k-mers seen t times or more */
    uint64_t assembly_windows;         /* every assembly's windows, junction windows included */
    uint64_t table_bytes;              /* the combined key table and the multiplicity table */
    uint64_t spectrum_table_bytes;     /* the read spectrum's largest table */
    uint64_t partitions, reruns;       /* of the read spectrum */
    float kernel_ms;                   /* CUDA events around every kernel, summed (0 under emulation) */
    float scan_ms, pack_ms, insert_ms, probe_ms, count_ms, assembly_ms;   /* record scan, read packing, assembly pack and claim, probes,
                                                                             spectrum count and histogram, every assembly's passes */
    double read_ms;                    /* host: reading and gunzipping the reads */
    double copy_ms;                    /* host wall time of the window uploads */
} ac_qv_info;
int ac_qv_dir(const char* reads, const char* const* inputs, uint32_t n_inputs, const char* out_dir, uint32_t k, const uint32_t* min_count,
              int32_t device, int32_t verbose, uint64_t* kmers, uint64_t* unsupported, uint64_t* solid_found, uint64_t cap, ac_qv_info* info);

/* `autocycler unassembled -r reads -i assemblies... -o out_dir [--kmer 21] [--min_count N] [--min_solid 100] [--min_fraction 0.5]`: the
 * reads the assembly does not explain, and the depth of the sequence it misses, counted on the GPU.  Not in the reference (DESIGN.md
 * section 21).  inputs: n_inputs paths, each a FASTA file or a directory, expanded as in ac_qv_dir; the contigs of all of them together are
 * the assembly, and A is the set of their canonical keys (qv's contig windows, junction windows included).  Read windows, r(key) and the
 * histogram are genome_size's; the solid threshold t is *min_count (1 .. AC_GENOME_SIZE_BINS - 1, else AC_EINPUT) or the valley when
 * min_count is NULL (no valley: AC_EINPUT "no k-mer depth peak: ...").  Per read i: s_i = its windows whose key has r >= t, a_i = those
 * of them whose key is not in A; the read is scored when s_i >= min_solid (>= 1, else AC_EINPUT) and selected when it is scored and
 * (double)a_i >= min_fraction * (double)s_i (0 < min_fraction <= 1, else AC_EINPUT).  The absent keys are the distinct keys with r >= t
 * not in A.  out_dir (created if needed) gets unassembled.fastq (the selected records in input order), unassembled.tsv,
 * fraction_histogram.tsv, absent_histogram.tsv, kmer_histogram.tsv (as helper genome_size -d writes it) and summary.tsv.  k: odd, 11..31,
 * else AC_EINPUT.  An assembly without windows (naming the inputs), reads without windows: AC_EINPUT.  The assembly set, the per-read
 * counters and the word indices beyond half the free device memory: AC_ERANGE.  verbose prints the settings and the counts to stderr.
 * Calls on one device run one at a time, with subsample's.  info may be NULL. */
typedef struct {
    uint64_t assemblies, contigs;
    uint32_t k;
    uint32_t min_count;                /* t, given or the valley */
    uint64_t valley;                   /* v of the reads' histogram (0: none) */
    uint64_t reads, read_windows, read_bases;
    uint64_t distinct;                 /* distinct canonical read k-mers */
    uint64_t scored_reads, selected_reads, selected_bases;
    uint64_t absent_kmers;             /* distinct keys with r >= t that the assembly lacks */
    double absent_median;              /* the median of their bins (NaN: no absent key) */
    double peak;                       /* genome_size's refined peak p* (NaN: the rule refuses the histogram) */
    double absent_copy_ratio;          /* absent_median / peak (NaN when either is) */
    uint64_t assembly_windows;         /* the assembly's windows, junction windows included */
    uint64_t table_bytes;              /* the assembly set */
    uint64_t read_bytes;               /* the per-read counters and lengths, and the word indices */
    uint64_t spectrum_table_bytes;     /* the read spectrum's largest table */
    uint64_t partitions, reruns;       /* of the read spectrum, over both sweeps */
    uint64_t read_passes;              /* 1, or 2 when the selected reads were gathered from a second read of the file */
    float kernel_ms;                   /* CUDA events around every kernel, summed (0 under emulation) */
    float scan_ms, pack_ms, claim_ms, count_ms, sweep_ms, gather_ms;   /* record scans, read packing and word indices, assembly pack and
                                                                          claim, spectrum count and histogram, attribution sweep (its
                                                                          recounts included), the FASTQ gather (with
                                                                          the second read's record scans) */
    double read_ms;                    /* host: reading and gunzipping the reads, both passes */
    double copy_ms;                    /* host wall time of the window uploads */
    double write_ms;                   /* host: writing the output files */
} ac_unassembled_info;
int ac_unassembled_dir(const char* reads, const char* const* inputs, uint32_t n_inputs, const char* out_dir, uint32_t k, const uint32_t* min_count,
                       uint64_t min_solid, double min_fraction, int32_t device, int32_t verbose, ac_unassembled_info* info);

/* `autocycler polish -r reads -i assembly -o out_dir [--kmer 21] [--min_count N] [--max_indel 3] [--rounds 3]`: the consensus corrected
 * where the reads' k-mers do not support it, with candidate edits scored on the GPU.  Not in the reference (DESIGN.md section 22).
 * assembly: one FASTA file (gzipped or not, loaded as load_fasta does).  Contig windows, r(key), the histogram and the solid threshold t
 * (*min_count, 1 .. AC_GENOME_SIZE_BINS - 1, else AC_EINPUT; the valley when min_count is NULL) are ac_qv_dir's, on each round's sequence.
 * Each round: a locus is a maximal run [a, b] of window starts with r < t (cyclic on a circular contig), tried when window a-1 exists and
 * has r >= t (and a circular contig is at least 2k + 2 max_indel long); at p0 = a + k - 1 its 3 substitutions, deletions of 1 .. max_indel
 * bases and insertions of every string of 1 .. max_indel bases before p0 are scored by the minimum r over the k + s windows of the edited
 * sequence that cover the edit; a candidate passes when all of them are windows (inside a linear contig) with r >= t.  A unique best is
 * accepted; accepted edits whose spans [a, p0 + d + k) overlap a kept one's (ascending a) wait for the next round.  The rounds stop after
 * `rounds` (1..10, else AC_EINPUT) or at the first that applies no edit.  max_indel: 1..4, else AC_EINPUT.  out_dir (created if needed)
 * gets polished.fasta, edits.tsv, rounds.tsv, remaining.bed (qv's unsupported/1.bed of polished.fasta) and summary.tsv.  k: odd, 11..31,
 * else AC_EINPUT.  An assembly or reads without windows: AC_EINPUT.  The window table beyond half the free device memory, or one locus's
 * candidate table beyond half of what the read spectrum leaves: AC_ERANGE.  verbose prints the settings, the counts and one line per round
 * to stderr.  Calls on one device run one at a time, with subsample's.  info may be NULL. */
typedef struct {
    uint64_t contigs;
    uint32_t k;
    uint32_t min_count;                /* t, given or the valley */
    uint64_t valley;                   /* v of the reads' histogram (0: none) */
    uint64_t reads, read_windows, read_bases;
    uint64_t distinct;                 /* distinct canonical read k-mers */
    uint64_t kmers_before, unsupported_before, kmers_after, unsupported_after;   /* the input's and polished.fasta's K and E */
    uint64_t edits, rounds, loci;      /* applied edits, rounds run, loci over every round */
    uint64_t table_bytes;              /* the contigs' window table */
    uint64_t candidate_table_bytes;    /* the largest candidate table */
    uint64_t batches;                  /* candidate batches over every round */
    uint64_t spectrum_table_bytes;     /* the read spectrum's largest table */
    uint64_t partitions, reruns;       /* of the read spectrum, over the count and every sweep */
    float kernel_ms;                   /* CUDA events around every kernel, summed (0 under emulation) */
    float scan_ms, pack_ms, count_ms, contig_ms, fill_ms, recount_ms, candidate_ms, choose_ms;   /* record scan, read packing, spectrum count
                                                                                                    and histogram, contig pack and claim, read
                                                                                                    count fills and unsupported masks, the
                                                                                                    sweeps' recounts of partitions, candidate
                                                                                                    claims and scores, choices */
    double read_ms;                    /* host: reading and gunzipping the reads */
    double copy_ms;                    /* host wall time of the window uploads */
    double host_ms;                    /* host: loci, overlaps, edits and the contigs' packing */
    double write_ms;                   /* host: writing the output files */
} ac_polish_info;
int ac_polish_fasta(const char* reads, const char* assembly, const char* out_dir, uint32_t k, const uint32_t* min_count, uint32_t max_indel,
                    uint32_t rounds, int32_t device, int32_t verbose, ac_polish_info* info);

/* `autocycler variants -r reads -i assembly -o out_dir [--kmer 21] [--min_count N] [--max_indel 1] [--min_fraction 0.1]`: the alleles the
 * reads carry beside the consensus, with every position's alternatives screened on the GPU.  Not in the reference (DESIGN.md section 23).
 * Inputs, windows, r(key) and t (*min_count, 1 .. AC_GENOME_SIZE_BINS - 1, else AC_EINPUT; the valley when min_count is NULL) are
 * ac_polish_fasta's, on the input sequence only; t is the least count an alternative allele needs.  A position p is tried when it can be
 * polish's p0 with a = p - k + 1 (a linear contig: p >= k - 1; a circular one: every p when it is at least 2k + 2 max_indel long) and the
 * window that ends at p has k A/C/G/T bases.  S(p, b): the input's bases [p - k + 1, p) followed by b; p is screened when r(S(p, e)) >= t
 * for some e other than its base.  Its candidates are polish's (3 substitutions, deletions of 1 .. max_indel bases, insertions of every
 * string of 1 .. max_indel bases before p), each taken only in its rightmost form, where its first base e in the edited sequence at p
 * differs from the input's (a deletion of d: base p + d, cyclic, A/C/G/T; an insertion: its first base), and only when S(p, e) passes the
 * screen.  Such a candidate passes as in polish (every checked window a window inside a linear contig, with r >= t); alt = the least r over
 * its checked windows, ref = the least r over the input's windows that start at a .. p + d (0 for a missing one; d = 0 but for a deletion),
 * PK = its checked windows whose key the input holds (an indel's last one left out).  A variant: alt >= min_fraction * (alt + ref) in f64,
 * 0 < min_fraction <= 1 (else AC_EINPUT).  max_indel: 0..3, else AC_EINPUT.  out_dir (created if needed) gets variants.vcf (VCF 4.2, indels
 * left-aligned, AF = alt / (alt + ref), AK, RK, PK) and summary.tsv.  k: odd, 11..31, else AC_EINPUT.  An assembly or reads without
 * windows: AC_EINPUT.  The window table beyond half the free device memory, or one position's candidate table beyond half of what the read
 * spectrum leaves: AC_ERANGE.  verbose prints the settings and the counts to stderr.  Calls on one device run one at a time, with
 * subsample's.  info may be NULL. */
typedef struct {
    uint64_t contigs;
    uint32_t k;
    uint32_t min_count;                /* t, given or the valley */
    uint64_t valley;                   /* v of the reads' histogram (0: none) */
    uint64_t reads, read_windows, read_bases;
    uint64_t distinct;                 /* distinct canonical read k-mers */
    uint64_t kmers;                    /* the input's windows */
    uint64_t positions, screened, candidates;   /* tried positions, those with an alternative window at or above t, rightmost candidates
                                                   whose first window passes */
    uint64_t loci;                     /* positions whose candidates were scored */
    uint64_t passing, variants;        /* candidates that pass, and of them the rows of variants.vcf */
    uint64_t substitutions, insertions, deletions, paralog, alt_major;
    uint64_t table_bytes;              /* the input's window table */
    uint64_t candidate_table_bytes;    /* the largest candidate table */
    uint64_t batches;                  /* candidate batches */
    uint64_t spectrum_table_bytes;     /* the read spectrum's largest table */
    uint64_t partitions, reruns;       /* of the read spectrum, over the count and every sweep */
    float kernel_ms;                   /* CUDA events around every kernel, summed (0 under emulation) */
    float scan_ms, pack_ms, count_ms, contig_ms, fill_ms, screen_ms, recount_ms, candidate_ms, ref_ms;   /* record scan, read packing,
                                                                                                    spectrum count and histogram, contig pack
                                                                                                    and claim, read count fills, the screen,
                                                                                                    the sweeps' recounts of partitions,
                                                                                                    candidate claims and scores, ref and PK */
    double read_ms;                    /* host: reading and gunzipping the reads */
    double copy_ms;                    /* host wall time of the window uploads */
    double host_ms;                    /* host: the contigs' packing, the candidates from the masks, the fraction test and left-alignment */
    double write_ms;                   /* host: writing the output files */
} ac_variants_info;
int ac_variants_fasta(const char* reads, const char* assembly, const char* out_dir, uint32_t k, const uint32_t* min_count, uint32_t max_indel,
                      double min_fraction, int32_t device, int32_t verbose, ac_variants_info* info);

#ifdef __cplusplus
}
#endif
#endif
