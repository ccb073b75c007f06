"""Host-side mirror of the reference's interface for the compress path, over the C ABI of
libautocycler_gpu.so (include/autocycler_gpu.h).

Names and argument meaning follow the reference (rrwick/Autocycler v0.6.1):
    KmerGraph(k_size).add_sequences(seqs, assembly_count)      kmer_graph.rs:79-90
    UnitigGraph.from_kmer_graph(kmer_graph)                    unitig_graph.rs:36-48
    simplify_structure(unitig_graph, seqs)                     graph_simplification.rs:26-40
    unitig_graph.save_gfa(path, seqs)                          unitig_graph.rs:317-331
    load_sequences(assemblies_dir, k_size, max_contigs)        compress.rs:98-133
    compress(assemblies_dir, autocycler_dir, k_size, ...)      compress.rs:32-50
    trim_path_start_end / _hairpin_start / _hairpin_end         trim.rs:288-326 (batch forms over lists of paths)
    unitig_graph.trim(min_identity, max_unitigs, mad)          trim.rs:43-51 (trim minus the file I/O)
    trim(cluster_dir, min_identity, max_unitigs, mad, ...)     trim.rs:36-53
    trim_dirs([cluster_dir, ...]) / resolve_dirs([...])        the same for several clusters, one device call per round
    bridge_best_paths(groups, weights)                         resolve.rs:430-462 (Bridge::new for a batch of bridges)
    unitig_graph.resolve() / resolve_text() / resolve_stats()   resolve.rs:41-67 (resolve minus the file I/O)
    resolve(cluster_dir), combine(autocycler_dir, in_gfas)      resolve.rs:31-69, combine.rs:25-49
    dotplot_rgb(seqs, res, kmer) / dotplot(input, out_png)      dotplot.rs:179-221 / dotplot.rs:44-52

There is no CPU path here: if the CUDA library is missing, or no device is present, every entry
point raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, "libautocycler_gpu.so")

AC_OK = 0


class AutocyclerGpuError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(f"[{code}] {message}")
        self.code = code
        self.message = message


class AcConfig(C.Structure):
    _fields_ = [("k", C.c_uint32), ("device", C.c_int32), ("stream", C.c_void_p), ("keep_positions", C.c_uint32),
                ("n_devices", C.c_int32), ("devices", C.POINTER(C.c_int32))]


class AcCounts(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("n_kmers", "n_unitigs", "n_links", "total_length", "seq_bytes", "n_fwd_pos",
                                         "n_rev_pos", "n_next", "n_sequences", "n_path_steps", "length_before_simplify")]


class AcUnitigs(C.Structure):
    _fields_ = [("number", C.POINTER(C.c_uint32)), ("seq_off", C.POINTER(C.c_uint64)), ("seq", C.POINTER(C.c_uint8)),
                ("depth", C.POINTER(C.c_double)),
                ("fpos_off", C.POINTER(C.c_uint64)), ("fpos", C.POINTER(C.c_uint32)), ("fpos_id_strand", C.POINTER(C.c_uint16)),
                ("rpos_off", C.POINTER(C.c_uint64)), ("rpos", C.POINTER(C.c_uint32)), ("rpos_id_strand", C.POINTER(C.c_uint16)),
                ("next_off", C.POINTER(C.c_uint64)), ("next", C.POINTER(C.c_int32))]


class AcTimings(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("h2d", "pack", "insert", "adjacency", "boundaries", "runs", "unitigs", "links", "seed_sort", "emit", "d2h",
                                        "device_total", "host_graph", "host_simplify", "host_gfa", "sample", "device_simplify", "device_gfa", "insert_kernel", "trim_kernel")] + \
               [(n, C.c_uint64) for n in ("insert_occurrences", "table_capacity", "table_used", "kernel_launches", "h2d_bytes", "d2h_bytes")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class AcResolveInfo(C.Structure):
    _fields_ = [("anchors", C.c_uint32), ("unique_bridges", C.c_uint32), ("conflicting_bridges", C.c_uint32), ("culled_bridges", C.c_uint32),
                ("jobs", C.c_uint64), ("cells", C.c_uint64), ("longest_path", C.c_uint64), ("shared_jobs", C.c_uint32), ("hbm_jobs", C.c_uint32),
                ("kernel_ms", C.c_float)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class AcBatchInfo(C.Structure):
    _fields_ = [("clusters", C.c_uint32), ("launches", C.c_uint32), ("jobs", C.c_uint64), ("cells", C.c_uint64), ("buffer_bytes", C.c_uint64),
                ("kernel_ms", C.c_float)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class AcDotplotInfo(C.Structure):
    _fields_ = [("windows", C.c_uint64), ("groups", C.c_uint64), ("dots", C.c_uint64), ("host_windows", C.c_uint64),
                ("bp_per_pixel", C.c_double), ("text_height", C.c_float), ("kernel_ms", C.c_float)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class AcSubsampleInfo(C.Structure):
    _fields_ = [("genome_size", C.c_uint64), ("reads_per_subset", C.c_uint64), ("input_count", C.c_uint64), ("input_bases", C.c_uint64),
                ("input_n50", C.c_uint64), ("windows", C.c_uint64), ("bytes_scanned", C.c_uint64), ("kernel_ms", C.c_float),
                ("read_ms", C.c_double), ("shuffle_ms", C.c_double), ("write_ms", C.c_double), ("copy_ms", C.c_double)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class AcGenomeSizeInfo(C.Structure):
    _fields_ = [("estimate", C.c_uint64), ("k", C.c_uint32), ("reruns", C.c_uint32), ("reads", C.c_uint64), ("bases", C.c_uint64),
                ("windows", C.c_uint64), ("distinct", C.c_uint64), ("valley", C.c_uint64), ("peak", C.c_uint64), ("peak_refined", C.c_double),
                ("solid", C.c_uint64), ("partitions", C.c_uint64), ("table_bytes", C.c_uint64), ("kernel_ms", C.c_float),
                ("scan_ms", C.c_float), ("pack_ms", C.c_float), ("count_ms", C.c_float), ("hist_ms", C.c_float), ("read_ms", C.c_double),
                ("copy_ms", C.c_double)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


GENOME_SIZE_BINS = 16384    # AC_GENOME_SIZE_BINS


class AcDepthInfo(C.Structure):
    _fields_ = [("contigs", C.c_uint64), ("unique_kmers", C.c_uint64), ("assembly_windows", C.c_uint64), ("reads", C.c_uint64),
                ("read_windows", C.c_uint64), ("read_bases", C.c_uint64), ("table_bytes", C.c_uint64), ("kept", C.c_uint64),
                ("k", C.c_uint32), ("filtered", C.c_int32), ("kernel_ms", C.c_float), ("scan_ms", C.c_float), ("pack_ms", C.c_float),
                ("insert_ms", C.c_float), ("probe_ms", C.c_float), ("median_ms", C.c_float), ("read_ms", C.c_double), ("copy_ms", C.c_double)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}

class AcQvInfo(C.Structure):
    _fields_ = [("assemblies", C.c_uint64), ("contigs", C.c_uint64), ("k", C.c_uint32), ("min_count", C.c_uint32), ("valley", C.c_uint64),
                ("reads", C.c_uint64), ("read_windows", C.c_uint64), ("read_bases", C.c_uint64), ("distinct", C.c_uint64),
                ("solid_kmers", C.c_uint64), ("assembly_windows", C.c_uint64), ("table_bytes", C.c_uint64), ("spectrum_table_bytes", C.c_uint64),
                ("partitions", C.c_uint64), ("reruns", C.c_uint64), ("kernel_ms", C.c_float), ("scan_ms", C.c_float), ("pack_ms", C.c_float),
                ("insert_ms", C.c_float), ("probe_ms", C.c_float), ("count_ms", C.c_float), ("assembly_ms", C.c_float), ("read_ms", C.c_double),
                ("copy_ms", C.c_double)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class AcUnassembledInfo(C.Structure):
    _fields_ = [("assemblies", C.c_uint64), ("contigs", C.c_uint64), ("k", C.c_uint32), ("min_count", C.c_uint32), ("valley", C.c_uint64),
                ("reads", C.c_uint64), ("read_windows", C.c_uint64), ("read_bases", C.c_uint64), ("distinct", C.c_uint64),
                ("scored_reads", C.c_uint64), ("selected_reads", C.c_uint64), ("selected_bases", C.c_uint64), ("absent_kmers", C.c_uint64),
                ("absent_median", C.c_double), ("peak", C.c_double), ("absent_copy_ratio", C.c_double), ("assembly_windows", C.c_uint64),
                ("table_bytes", C.c_uint64), ("read_bytes", C.c_uint64), ("spectrum_table_bytes", C.c_uint64), ("partitions", C.c_uint64),
                ("reruns", C.c_uint64), ("read_passes", C.c_uint64), ("kernel_ms", C.c_float), ("scan_ms", C.c_float), ("pack_ms", C.c_float),
                ("claim_ms", C.c_float), ("count_ms", C.c_float), ("sweep_ms", C.c_float), ("gather_ms", C.c_float), ("read_ms", C.c_double),
                ("copy_ms", C.c_double), ("write_ms", C.c_double)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class AcPolishInfo(C.Structure):
    _fields_ = [("contigs", C.c_uint64), ("k", C.c_uint32), ("min_count", C.c_uint32), ("valley", C.c_uint64), ("reads", C.c_uint64),
                ("read_windows", C.c_uint64), ("read_bases", C.c_uint64), ("distinct", C.c_uint64), ("kmers_before", C.c_uint64),
                ("unsupported_before", C.c_uint64), ("kmers_after", C.c_uint64), ("unsupported_after", C.c_uint64), ("edits", C.c_uint64),
                ("rounds", C.c_uint64), ("loci", C.c_uint64), ("table_bytes", C.c_uint64), ("candidate_table_bytes", C.c_uint64),
                ("batches", C.c_uint64), ("spectrum_table_bytes", C.c_uint64), ("partitions", C.c_uint64), ("reruns", C.c_uint64),
                ("kernel_ms", C.c_float), ("scan_ms", C.c_float), ("pack_ms", C.c_float), ("count_ms", C.c_float), ("contig_ms", C.c_float),
                ("fill_ms", C.c_float), ("recount_ms", C.c_float), ("candidate_ms", C.c_float), ("choose_ms", C.c_float),
                ("read_ms", C.c_double), ("copy_ms", C.c_double), ("host_ms", C.c_double), ("write_ms", C.c_double)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class AcVariantsInfo(C.Structure):
    _fields_ = [("contigs", C.c_uint64), ("k", C.c_uint32), ("min_count", C.c_uint32), ("valley", C.c_uint64), ("reads", C.c_uint64),
                ("read_windows", C.c_uint64), ("read_bases", C.c_uint64), ("distinct", C.c_uint64), ("kmers", C.c_uint64),
                ("positions", C.c_uint64), ("screened", C.c_uint64), ("candidates", C.c_uint64), ("loci", C.c_uint64), ("passing", C.c_uint64),
                ("variants", C.c_uint64), ("substitutions", C.c_uint64), ("insertions", C.c_uint64), ("deletions", C.c_uint64),
                ("paralog", C.c_uint64), ("alt_major", C.c_uint64), ("table_bytes", C.c_uint64), ("candidate_table_bytes", C.c_uint64),
                ("batches", C.c_uint64), ("spectrum_table_bytes", C.c_uint64), ("partitions", C.c_uint64), ("reruns", C.c_uint64),
                ("kernel_ms", C.c_float), ("scan_ms", C.c_float), ("pack_ms", C.c_float), ("count_ms", C.c_float), ("contig_ms", C.c_float),
                ("fill_ms", C.c_float), ("screen_ms", C.c_float), ("recount_ms", C.c_float), ("candidate_ms", C.c_float), ("ref_ms", C.c_float),
                ("read_ms", C.c_double), ("copy_ms", C.c_double), ("host_ms", C.c_double), ("write_ms", C.c_double)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


EXPORTS = ["ac_last_error", "ac_version", "ac_create", "ac_destroy", "ac_add_sequence", "ac_clear_sequences", "ac_upload",
           "ac_build", "ac_compress", "ac_simplify", "ac_merge_linear_paths", "ac_renumber_unitigs", "ac_load_gfa", "ac_bind_host_to_device", "ac_decompress_gfa", "ac_pairwise_distances", "ac_distance_matrix_text", "ac_sequence_reconstruct", "ac_counts_get", "ac_unitigs_copy", "ac_path_copy", "ac_gfa_size", "ac_gfa_copy",
           "ac_timings_get", "ac_compress_dir", "ac_compress_dir_devices", "ac_load_sequences", "ac_sequence_get",
           "ac_build_local", "ac_entries_count", "ac_entries_export", "ac_entries_merge", "ac_runs_local", "ac_runs_export",
           "ac_runs_import", "ac_runs_import_padded", "ac_build_finish", "ac_compress_finish", "ac_gfa_data",
           "ac_compress_finish_split", "ac_path_tokens_export", "ac_path_lines_render", "ac_path_lines_data", "ac_upload_shard", "ac_strand_block",
           "ac_trim_paths", "ac_trim", "ac_trim_yaml", "ac_trim_stats", "ac_trim_dir", "ac_trim_dirs",
           "ac_cluster", "ac_cluster_text", "ac_cluster_assignments", "ac_cluster_stats", "ac_upgma", "ac_cluster_dir",
           "ac_bridge_best_paths", "ac_resolve", "ac_resolve_text", "ac_resolve_stats", "ac_resolve_dir", "ac_resolve_dirs", "ac_combine_dir",
           "ac_dotplot_rgb", "ac_dotplot_dir", "ac_png_write",
           "ac_clean_gfa", "ac_clean_text", "ac_gfa_to_fasta", "ac_gfa_fasta_text", "ac_table_text",
           "ac_subsample_dir", "ac_genome_size", "ac_subsample_words", "ac_subsample_shuffle",
           "ac_genome_size_estimate", "ac_genome_size_from_histogram",
           "ac_depth_fasta", "ac_depth_filter_text", "ac_depth_from_header", "ac_qv_dir", "ac_unassembled_dir",
           "ac_polish_fasta", "ac_variants_fasta"]

_libs = {}


def _raise_unless_ok(lib, rc):
    """Raises the library's error for a call without a handle."""
    if rc != AC_OK:
        raise AutocyclerGpuError(rc, lib.ac_last_error(None).decode())


def _weight_list(weights):
    """{unitig: length} or a list indexed by unitig number -> the list the C ABI takes."""
    if not isinstance(weights, dict):
        return list(weights)
    w = [0] * (max(weights) + 1 if weights else 1)
    for u, ln in weights.items():
        w[u] = ln
    return w


def load_library(path=None):
    """Loads the C-ABI library (default: the in-tree CUDA build) and declares its prototypes."""
    path = os.path.abspath(path or DEFAULT_LIB)
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise AutocyclerGpuError(-2, f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                                     "(the GPU path has no CPU fallback)")
    lib = C.CDLL(path)
    lib.ac_last_error.restype = C.c_char_p
    lib.ac_last_error.argtypes = [C.c_void_p]
    lib.ac_version.restype = C.c_char_p
    lib.ac_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(AcConfig)]
    lib.ac_destroy.argtypes = [C.c_void_p]
    lib.ac_destroy.restype = None
    lib.ac_add_sequence.argtypes = [C.c_void_p, C.c_uint16, C.c_char_p, C.c_uint64, C.c_char_p, C.c_char_p]
    lib.ac_clear_sequences.argtypes = [C.c_void_p]
    for name in ("ac_upload", "ac_build", "ac_compress", "ac_simplify", "ac_renumber_unitigs"):
        getattr(lib, name).argtypes = [C.c_void_p]
    lib.ac_merge_linear_paths.argtypes = [C.c_void_p, C.c_int]
    lib.ac_load_gfa.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64]
    lib.ac_bind_host_to_device.argtypes = [C.c_int32]
    lib.ac_pairwise_distances.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.c_uint64]
    lib.ac_distance_matrix_text.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.ac_decompress_gfa.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int32, C.c_int32]
    lib.ac_sequence_reconstruct.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.ac_counts_get.argtypes = [C.c_void_p, C.POINTER(AcCounts)]
    lib.ac_unitigs_copy.argtypes = [C.c_void_p, C.POINTER(AcUnitigs)]
    lib.ac_path_copy.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_int32), C.c_uint64, C.POINTER(C.c_uint64)]
    lib.ac_gfa_size.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    lib.ac_gfa_copy.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    lib.ac_timings_get.argtypes = [C.c_void_p, C.POINTER(AcTimings)]
    lib.ac_compress_dir.argtypes = [C.c_char_p, C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32, C.c_int32]
    lib.ac_compress_dir_devices.argtypes = [C.c_char_p, C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_int32), C.c_int32, C.c_int32]
    lib.ac_load_sequences.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64)]
    lib.ac_sequence_get.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_uint16), C.POINTER(C.c_uint64), C.c_char_p, C.c_uint64,
                                    C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64]
    lib.ac_build_local.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
    lib.ac_entries_count.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    lib.ac_entries_export.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    lib.ac_entries_merge.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    lib.ac_runs_local.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    lib.ac_runs_export.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    lib.ac_runs_import.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    lib.ac_runs_import_padded.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_uint32]
    lib.ac_build_finish.argtypes = [C.c_void_p]
    lib.ac_compress_finish.argtypes = [C.c_void_p]
    lib.ac_compress_finish_split.argtypes = [C.c_void_p]
    lib.ac_upload_shard.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    lib.ac_strand_block.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    lib.ac_path_tokens_export.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_uint32]
    lib.ac_path_lines_render.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    lib.ac_path_lines_data.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    lib.ac_gfa_data.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    lib.ac_trim_paths.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(C.c_uint32),
                                  C.c_uint64, C.c_double, C.c_uint32, C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.POINTER(C.c_uint8)]
    lib.ac_trim.argtypes = [C.c_void_p, C.c_double, C.c_uint32, C.c_double]
    lib.ac_trim_yaml.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.ac_trim_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]
    lib.ac_trim_dir.argtypes = [C.c_char_p, C.c_double, C.c_uint32, C.c_double, C.c_uint32, C.c_int32, C.c_int32]
    lib.ac_trim_dirs.argtypes = [C.POINTER(C.c_char_p), C.c_uint32, C.c_double, C.c_uint32, C.c_double, C.c_uint32, C.c_int32, C.c_int32,
                                 C.POINTER(AcBatchInfo)]
    lib.ac_cluster.argtypes = [C.c_void_p, C.c_double, C.c_int64, C.POINTER(C.c_uint16), C.c_uint64]
    lib.ac_cluster_text.argtypes = [C.c_void_p, C.c_int32, C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.ac_cluster_assignments.argtypes = [C.c_void_p, C.POINTER(C.c_uint16), C.POINTER(C.c_uint8), C.c_uint64]
    lib.ac_cluster_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_float),
                                     C.POINTER(C.c_float), C.POINTER(C.c_double)]
    lib.ac_upgma.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                             C.POINTER(C.c_uint32), C.POINTER(C.c_double)]
    lib.ac_cluster_dir.argtypes = [C.c_char_p, C.c_double, C.c_int64, C.c_uint32, C.c_char_p, C.c_int32, C.c_int32]
    lib.ac_bridge_best_paths.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(C.c_uint64), C.c_uint64,
                                         C.POINTER(C.c_uint32), C.c_uint64, C.POINTER(C.c_uint32), C.POINTER(C.c_int32), C.POINTER(C.c_uint64)]
    lib.ac_resolve.argtypes = [C.c_void_p, C.c_int32]
    lib.ac_resolve_text.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.ac_resolve_stats.argtypes = [C.c_void_p, C.POINTER(AcResolveInfo)]
    lib.ac_resolve_dir.argtypes = [C.c_char_p, C.c_int32, C.c_int32]
    lib.ac_resolve_dirs.argtypes = [C.POINTER(C.c_char_p), C.c_uint32, C.c_int32, C.c_int32, C.POINTER(AcBatchInfo)]
    lib.ac_combine_dir.argtypes = [C.c_char_p, C.POINTER(C.c_char_p), C.c_uint32, C.c_int32]
    lib.ac_dotplot_rgb.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_uint64), C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.c_uint32,
                                   C.c_uint32, C.c_uint32, C.c_char_p, C.c_int32, C.c_void_p, C.POINTER(AcDotplotInfo)]
    lib.ac_dotplot_dir.argtypes = [C.c_char_p, C.c_char_p, C.c_uint32, C.c_uint32, C.c_char_p, C.c_int32, C.c_int32, C.POINTER(AcDotplotInfo)]
    lib.ac_png_write.argtypes = [C.c_char_p, C.c_void_p, C.c_uint32, C.c_uint32]
    lib.ac_clean_gfa.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(C.c_double), C.c_int32]
    lib.ac_clean_text.argtypes = [C.c_char_p, C.c_uint64, C.POINTER(C.c_uint32), C.c_uint64, C.POINTER(C.c_uint32), C.c_uint64,
                                  C.POINTER(C.c_double), C.c_int32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.ac_gfa_to_fasta.argtypes = [C.c_char_p, C.c_char_p, C.c_int32]
    lib.ac_gfa_fasta_text.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.ac_subsample_dir.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint64, C.c_double, C.c_uint64, C.c_int32, C.c_int32,
                                     C.POINTER(AcSubsampleInfo)]
    lib.ac_genome_size.argtypes = [C.c_char_p, C.POINTER(C.c_uint64)]
    lib.ac_subsample_words.argtypes = [C.c_uint64, C.c_uint32, C.POINTER(C.c_uint32), C.c_uint64]
    lib.ac_subsample_shuffle.argtypes = [C.c_uint64, C.c_uint64, C.POINTER(C.c_uint32)]
    lib.ac_genome_size_estimate.argtypes = [C.c_char_p, C.c_uint32, C.c_int32, C.c_char_p, C.c_int32, C.POINTER(C.c_uint64),
                                            C.POINTER(AcGenomeSizeInfo)]
    lib.ac_genome_size_from_histogram.argtypes = [C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(AcGenomeSizeInfo)]
    lib.ac_depth_fasta.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int32, C.c_uint32, C.POINTER(C.c_double),
                                   C.POINTER(C.c_double), C.c_int32, C.c_int32, C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.c_uint64,
                                   C.POINTER(AcDepthInfo)]
    lib.ac_depth_filter_text.argtypes = [C.c_char_p, C.c_uint64, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_void_p, C.c_uint64,
                                         C.POINTER(C.c_uint64)]
    lib.ac_depth_from_header.argtypes = [C.c_char_p, C.POINTER(C.c_double)]
    lib.ac_qv_dir.argtypes = [C.c_char_p, C.POINTER(C.c_char_p), C.c_uint32, C.c_char_p, C.c_uint32, C.POINTER(C.c_uint32), C.c_int32, C.c_int32,
                              C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(AcQvInfo)]
    lib.ac_unassembled_dir.argtypes = [C.c_char_p, C.POINTER(C.c_char_p), C.c_uint32, C.c_char_p, C.c_uint32, C.POINTER(C.c_uint32), C.c_uint64,
                                       C.c_double, C.c_int32, C.c_int32, C.POINTER(AcUnassembledInfo)]
    lib.ac_polish_fasta.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint32, C.POINTER(C.c_uint32), C.c_uint32, C.c_uint32, C.c_int32,
                                    C.c_int32, C.POINTER(AcPolishInfo)]
    lib.ac_variants_fasta.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint32, C.POINTER(C.c_uint32), C.c_uint32, C.c_double,
                                      C.c_int32, C.c_int32, C.POINTER(AcVariantsInfo)]
    lib.ac_table_text.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint64, C.c_int32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
    _libs[path] = lib
    return lib


class Sequence:
    """sequence.rs:19-28: the padded forward strand plus what save_gfa prints."""

    def __init__(self, id, forward_seq, filename, contig_header, length):
        self.id, self.forward_seq, self.filename, self.contig_header, self.length = id, forward_seq, filename, contig_header, length

    @staticmethod
    def new_with_seq(id, seq, filename, contig_header, length, half_k):   # sequence.rs:31-59
        if any(c not in "ACGT" for c in seq):
            raise AutocyclerGpuError(-6, f"{filename} contains non-ACGT characters")
        return Sequence(id, "." * half_k + seq + "." * half_k, filename, contig_header, length)


def stream_handle(stream):
    """The value of ac_config.stream for a caller's stream: None -> NULL (the library creates a private, non-blocking stream); a
    cudaStream_t -> itself; 0 — CUDA's legacy default stream, what torch.cuda.current_stream().cuda_stream is unless the caller switched
    streams — -> its explicit handle cudaStreamLegacy (0x1), because NULL already means "private"."""
    return None if stream is None else (int(stream) or 1)


class _Handle:
    def __init__(self, lib, k, device=0, stream=None, keep_positions=False, devices=None):
        self.lib = lib
        self.k = k
        self.stream = stream             # what the caller named (None: the library's own); stream_handle() is what the library is given
        self.ptr = C.c_void_p()
        devs = (C.c_int32 * len(devices))(*devices) if devices else None      # several GPUs driven by this one process (ac_config.n_devices)
        cfg = AcConfig(k, device, stream_handle(stream), 1 if keep_positions else 0, len(devices) if devices else 0, devs)
        _raise_unless_ok(lib, lib.ac_create(C.byref(self.ptr), C.byref(cfg)))

    def check(self, rc):
        if rc != AC_OK:
            raise AutocyclerGpuError(rc, self.lib.ac_last_error(self.ptr).decode())

    def runs_on(self, cuda_stream):
        """True when the library was told to run on exactly this cudaStream_t (then work a caller enqueues there is ordered with the
        library's by the stream itself); a handle with a private stream is ordered with nobody and needs the device to settle."""
        return self.stream is not None and int(self.stream) == int(cuda_stream)

    def close(self):
        if self.ptr:
            self.lib.ac_destroy(self.ptr)
            self.ptr = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class KmerGraph:
    """kmer_graph.rs:73-90.  The k-mers live in a hash table in HBM; `add_sequences` stages and uploads the strands,
    the table itself is built by UnitigGraph.from_kmer_graph (one fused device pipeline)."""

    def __init__(self, k_size, device=0, stream=None, lib=None, keep_positions=False, devices=None):
        self.k_size = k_size
        self._h = _Handle(lib or load_library(), k_size, device, stream, keep_positions, devices)
        self.assembly_count = 0
        self.sequences = []

    def add_sequences(self, seqs, assembly_count, upload=True):
        h = self._h
        h.check(h.lib.ac_clear_sequences(h.ptr))
        for s in seqs:
            fwd = s.forward_seq if isinstance(s.forward_seq, bytes) else s.forward_seq.encode()
            h.check(h.lib.ac_add_sequence(h.ptr, s.id, fwd, len(fwd), s.filename.encode(), s.contig_header.encode()))
        self.assembly_count = assembly_count
        self.sequences = list(seqs)
        if upload:
            self.upload()

    def upload(self):
        self._h.check(self._h.lib.ac_upload(self._h.ptr))


class UnitigGraph:
    """unitig_graph.rs:28-48."""

    def __init__(self, kmer_graph):
        self._kg = kmer_graph
        self._h = kmer_graph._h
        self.k_size = kmer_graph.k_size

    @staticmethod
    def from_kmer_graph(kmer_graph):
        g = UnitigGraph(kmer_graph)
        g._h.check(g._h.lib.ac_build(g._h.ptr))
        return g

    @staticmethod
    def compress(kmer_graph):
        """compress.rs:42-47 as one device pipeline (ac_compress): the simplified, renumbered graph; its GFA text is ready
        (gfa_view / gfa_bytes / save_gfa), the graph arrays are fetched from HBM when first asked for."""
        g = UnitigGraph(kmer_graph)
        g._h.check(g._h.lib.ac_compress(g._h.ptr))
        return g

    @staticmethod
    def from_gfa_lines(gfa_lines, lib=None, device=0):   # unitig_graph.rs:55-74 -> (UnitigGraph, [Sequence without bytes])
        text = gfa_lines if isinstance(gfa_lines, (bytes, str)) else "\n".join(l.rstrip("\n") for l in gfa_lines) + "\n"
        text = text.encode() if isinstance(text, str) else text
        kg = KmerGraph(51, device=device, lib=lib)          # the handle's k is replaced by the file's KM:i: value
        g = UnitigGraph(kg)
        g._h.check(g._h.lib.ac_load_gfa(g._h.ptr, text, len(text)))
        g.k_size = None
        seqs = []
        n = g.counts().n_sequences
        for i in range(n):
            sid, ln = C.c_uint16(), C.c_uint64()
            fn, hd = C.create_string_buffer(4096), C.create_string_buffer(65536)
            g._h.check(g._h.lib.ac_sequence_get(g._h.ptr, i, C.byref(sid), C.byref(ln), None, 0, fn, len(fn), hd, len(hd)))
            seqs.append(Sequence(sid.value, None, fn.value.decode(), hd.value.decode(), ln.value))
        return g, seqs

    @staticmethod
    def from_gfa_file(gfa_filename, lib=None, device=0):   # unitig_graph.rs:50-53
        with open(gfa_filename, "rb") as f:
            return UnitigGraph.from_gfa_lines(f.read(), lib=lib, device=device)

    def counts(self):
        c = AcCounts()
        self._h.check(self._h.lib.ac_counts_get(self._h.ptr, C.byref(c)))
        return c

    def kmer_count(self):           # KmerGraph.kmers.len(), compress.rs:152
        return self.counts().n_kmers

    def total_length(self):         # unitig_graph.rs:474-476
        return self.counts().total_length

    def link_count(self):           # unitig_graph.rs:478-507 (.1)
        return self.counts().n_links

    def timings(self):
        t = AcTimings()
        self._h.check(self._h.lib.ac_timings_get(self._h.ptr, C.byref(t)))
        return t

    def unitigs(self, positions=False):
        """-> list of dicts (number, seq, depth, forward_next, reverse_next[, forward_positions, reverse_positions])
        in the graph's current order."""
        c = self.counts()
        U = c.n_unitigs
        number = (C.c_uint32 * U)(); seq_off = (C.c_uint64 * (U + 1))(); seq = (C.c_uint8 * max(1, c.seq_bytes))()
        depth = (C.c_double * U)(); next_off = (C.c_uint64 * (2 * U + 1))(); nxt = (C.c_int32 * max(1, c.n_next))()
        u = AcUnitigs()
        u.number = number; u.seq_off = seq_off; u.seq = seq; u.depth = depth; u.next_off = next_off; u.next = nxt
        if positions:
            fo = (C.c_uint64 * (U + 1))(); fp = (C.c_uint32 * max(1, c.n_fwd_pos))(); fi = (C.c_uint16 * max(1, c.n_fwd_pos))()
            ro = (C.c_uint64 * (U + 1))(); rp = (C.c_uint32 * max(1, c.n_rev_pos))(); ri = (C.c_uint16 * max(1, c.n_rev_pos))()
            u.fpos_off = fo; u.fpos = fp; u.fpos_id_strand = fi; u.rpos_off = ro; u.rpos = rp; u.rpos_id_strand = ri
        self._h.check(self._h.lib.ac_unitigs_copy(self._h.ptr, C.byref(u)))
        raw = bytes(seq)
        out = []
        for i in range(U):
            d = {"number": number[i], "seq": raw[seq_off[i]:seq_off[i + 1]].decode(), "depth": depth[i],
                 "forward_next": [nxt[x] for x in range(next_off[2 * i], next_off[2 * i + 1])],
                 "reverse_next": [nxt[x] for x in range(next_off[2 * i + 1], next_off[2 * i + 2])]}
            if positions:
                fmt = lambda p, t: f"{t & 0x7FFF}{'+' if t & 0x8000 else '-'}{p}"   # position.rs:54-58
                d["forward_positions"] = [fmt(fp[x], fi[x]) for x in range(fo[i], fo[i + 1])]
                d["reverse_positions"] = [fmt(rp[x], ri[x]) for x in range(ro[i], ro[i + 1])]
            out.append(d)
        return out

    def get_unitig_path_for_sequence_i32(self, seq_index):   # unitig_graph.rs:467-472
        n = C.c_uint64()
        self._h.check(self._h.lib.ac_path_copy(self._h.ptr, seq_index, None, 0, C.byref(n)))
        buf = (C.c_int32 * max(1, n.value))()
        self._h.check(self._h.lib.ac_path_copy(self._h.ptr, seq_index, buf, n.value, C.byref(n)))
        return list(buf[:n.value])

    def gfa_bytes(self):            # the bytes save_gfa writes
        n = C.c_uint64()
        self._h.check(self._h.lib.ac_gfa_size(self._h.ptr, C.byref(n)))
        out = bytearray(n.value)
        if n.value:
            buf = (C.c_char * n.value).from_buffer(out)     # the library writes straight into the result, no second copy
            self._h.check(self._h.lib.ac_gfa_copy(self._h.ptr, buf, n.value))
            del buf
        return out

    def gfa_view(self):             # the same bytes without a copy: a memoryview of the library's buffer, valid until the next call on this graph
        n = C.c_uint64(); ptr = C.c_void_p()
        self._h.check(self._h.lib.ac_gfa_data(self._h.ptr, C.byref(ptr), C.byref(n)))
        return memoryview((C.c_char * n.value).from_address(ptr.value)) if n.value else memoryview(b"")

    def pairwise_contig_distances(self):   # cluster.rs:132-151 -> S x S list of lists (row a, column b)
        S = self.counts().n_sequences
        buf = (C.c_double * max(1, S * S))()
        self._h.check(self._h.lib.ac_pairwise_distances(self._h.ptr, buf, S * S))
        return [[buf[a * S + b] for b in range(S)] for a in range(S)]

    def _text(self, fn, *args):   # a two-call getter fn(handle, *args, out, cap, length): the length, then the text
        n = C.c_uint64()
        self._h.check(fn(self._h.ptr, *args, None, 0, C.byref(n)))
        buf = C.create_string_buffer(max(1, n.value))
        self._h.check(fn(self._h.ptr, *args, buf, n.value, C.byref(n)))
        return buf.raw[:n.value].decode()

    def distance_matrix_text(self):   # cluster.rs:160-176
        return self._text(self._h.lib.ac_distance_matrix_text)

    def renumber_unitigs(self):   # unitig_graph.rs:295-315
        self._h.check(self._h.lib.ac_renumber_unitigs(self._h.ptr))

    def reconstruct_original_sequence(self, index):   # unitig_graph.rs:383-388, by position in the sequence list
        return self._text(self._h.lib.ac_sequence_reconstruct, index)

    def trim(self, min_identity=0.75, max_unitigs=5000, mad=5.0):   # trim.rs:43-51 on this (loaded) graph
        """Start-end and hairpin trimming (alignments on the GPU), length outliers, clean-up: afterwards the graph and its sequences are
        2_trimmed.gfa's; trimmed_yaml() is 2_trimmed.yaml and timings().trim_kernel the alignment kernels' time."""
        self._h.check(self._h.lib.ac_trim(self._h.ptr, min_identity, max_unitigs, mad))

    def trimmed_yaml(self):   # TrimmedClusterMetrics (metrics.rs:209-225) after trim()
        return self._text(self._h.lib.ac_trim_yaml)

    def trim_stats(self):   # what the last trim aligned
        jobs, cells, path = C.c_uint64(), C.c_uint64(), C.c_uint64(); window = C.c_uint32()
        self._h.check(self._h.lib.ac_trim_stats(self._h.ptr, C.byref(jobs), C.byref(cells), C.byref(window), C.byref(path)))
        return {"alignments": jobs.value, "dp_cells": cells.value, "max_window": window.value, "max_path": path.value}

    def cluster(self, cutoff=0.2, min_assemblies=None, manual=None):   # cluster.rs:42-59 on this graph (loaded input_assemblies.gfa)
        """Distances and UPGMA on the GPU, then clustering, QC and the output texts: cluster_text() returns them, cluster_assignments()
        the per-sequence result and cluster_stats() the kernel times.  manual: node numbers of the tree (None: automatic)."""
        man = sorted(manual or [])
        arr = (C.c_uint16 * max(1, len(man)))(*man)
        self._h.check(self._h.lib.ac_cluster(self._h.ptr, float(cutoff), -1 if min_assemblies is None else int(min_assemblies), arr, len(man)))

    CLUSTER_TEXTS = {"phylip": 0, "newick": 1, "tsv": 2, "yaml": 3, "gfa": 4, "untrimmed_yaml": 5}

    def cluster_text(self, what, cluster=0):   # "phylip", "newick", "tsv", "yaml"; per cluster: "gfa", "untrimmed_yaml"
        return self._text(self._h.lib.ac_cluster_text, self.CLUSTER_TEXTS[what], cluster)

    def cluster_assignments(self, n_seqs):   # -> [(cluster number, passed QC)] per sequence
        cl = (C.c_uint16 * max(1, n_seqs))(); ps = (C.c_uint8 * max(1, n_seqs))()
        self._h.check(self._h.lib.ac_cluster_assignments(self._h.ptr, cl, ps, n_seqs))
        return [(cl[i], bool(ps[i])) for i in range(n_seqs)]

    def cluster_stats(self):
        n, p, f = C.c_uint32(), C.c_uint32(), C.c_uint32(); dm, um = C.c_float(), C.c_float(); gm = C.c_double()
        self._h.check(self._h.lib.ac_cluster_stats(self._h.ptr, C.byref(n), C.byref(p), C.byref(f), C.byref(dm), C.byref(um), C.byref(gm)))
        return {"sequences": n.value, "pass_clusters": p.value, "fail_clusters": f.value, "distance_ms": dm.value, "upgma_ms": um.value,
                "cluster_gfa_ms": gm.value}

    def resolve(self, verbose=False):   # resolve.rs:41-67 on this graph (a loaded 2_trimmed.gfa)
        """Anchors, bridges (their path distances on the GPU), the unique bridges applied, culling and the final bridges: resolve_text()
        returns 3_bridged.gfa, 4_merged.gfa and 5_final.gfa, resolve_stats() the counts and the kernel time.  The graph is unchanged."""
        self._h.check(self._h.lib.ac_resolve(self._h.ptr, 1 if verbose else 0))

    RESOLVE_TEXTS = {"bridged": 0, "merged": 1, "final": 2}

    def resolve_text(self, what):   # "bridged", "merged" or "final"
        return self._text(self._h.lib.ac_resolve_text, self.RESOLVE_TEXTS[what])

    def resolve_stats(self):
        info = AcResolveInfo()
        self._h.check(self._h.lib.ac_resolve_stats(self._h.ptr, C.byref(info)))
        return info.as_dict()

    def save_gfa(self, gfa_filename, sequences=None, use_other_colour=False):   # unitig_graph.rs:317-331
        with open(gfa_filename, "wb") as f:
            f.write(self.gfa_bytes())


def simplify_structure(graph, seqs=None):   # graph_simplification.rs:26-40
    graph._h.check(graph._h.lib.ac_simplify(graph._h.ptr))


def decompress(in_gfa, out_dir=None, out_file=None, lib=None, device=0):   # decompress.rs:27-38
    lib = lib or load_library()
    _raise_unless_ok(lib, lib.ac_decompress_gfa(os.fsencode(in_gfa), os.fsencode(out_dir) if out_dir else None,
                                                os.fsencode(out_file) if out_file else None, device, 0))


def merge_linear_paths(graph, seqs=()):   # graph_simplification.rs:315-371; seqs=None/[] merges without regard to the paths
    graph._h.check(graph._h.lib.ac_merge_linear_paths(graph._h.ptr, 1 if seqs is not None and len(seqs) else 0))


def load_sequences(assemblies_dir, k_size, max_contigs=25, threads=8, lib=None, device=0, stream=None):
    """compress.rs:98-133 -> (KmerGraph holding the staged sequences, [Sequence], assembly_count)."""
    kg = KmerGraph(k_size, device=device, lib=lib, stream=stream)
    h = kg._h
    count = C.c_uint64()
    h.check(h.lib.ac_load_sequences(h.ptr, os.fsencode(assemblies_dir), max_contigs, threads, C.byref(count)))
    seqs = []
    i = 0
    while True:
        sid = C.c_uint16(); length = C.c_uint64()
        if h.lib.ac_sequence_get(h.ptr, i, C.byref(sid), C.byref(length), None, 0, None, 0, None, 0) != AC_OK:
            break
        fwd = C.create_string_buffer(length.value + k_size); fn = C.create_string_buffer(4096); hd = C.create_string_buffer(1 << 16)
        h.check(h.lib.ac_sequence_get(h.ptr, i, None, None, fwd, len(fwd), fn, len(fn), hd, len(hd)))
        seqs.append(Sequence(sid.value, fwd.value.decode(), fn.value.decode(), hd.value.decode(), length.value))
        i += 1
    kg.sequences = seqs
    kg.assembly_count = count.value
    return kg, seqs, count.value


def compress(assemblies_dir, autocycler_dir, k_size=51, max_contigs=25, threads=8, device=0, verbose=False, lib=None, devices=None):
    """compress.rs:32-50: writes <autocycler_dir>/input_assemblies.gfa and .yaml.  devices=[...]: sharded by file over several GPUs."""
    lib = lib or load_library()
    devs = list(devices) if devices else [device]
    _raise_unless_ok(lib, lib.ac_compress_dir_devices(os.fsencode(assemblies_dir), os.fsencode(autocycler_dir), k_size, max_contigs, threads,
                                                      (C.c_int32 * len(devs))(*devs), len(devs), 1 if verbose else 0))


TRIM_START_END, TRIM_HAIRPIN_START, TRIM_HAIRPIN_END = 0, 1, 2


def _trim_paths(mode, paths, weights, min_identity, max_unitigs, lib=None, device=0, handle=None):
    """One trim.rs:288-326 trim of every path in `paths` (lists of signed unitig numbers); weights: {unitig: length} or a list indexed
    by unitig number.  -> [trimmed path or None]"""
    lib = lib or load_library()
    h = handle or _Handle(lib, 51, device)
    w = _weight_list(weights)
    flat = [u for p in paths for u in p]
    off = [0]
    for p in paths:
        off.append(off[-1] + len(p))
    n = len(paths)
    vals = (C.c_int32 * max(1, len(flat)))(*flat)
    out = (C.c_int32 * max(1, len(flat)))()
    out_off = (C.c_uint64 * (n + 1))()
    trimmed = (C.c_uint8 * max(1, n))()
    h.check(lib.ac_trim_paths(h.ptr, mode, vals, (C.c_uint64 * (n + 1))(*off), n, (C.c_uint32 * max(1, len(w)))(*w), len(w),
                              float(min_identity), max_unitigs, out, out_off, trimmed))
    return [list(out[out_off[x]:out_off[x + 1]]) if trimmed[x] else None for x in range(n)]


def trim_path_start_end(paths, weights, min_identity, max_unitigs, **kw):      # trim.rs:288-296
    return _trim_paths(TRIM_START_END, paths, weights, min_identity, max_unitigs, **kw)


def trim_path_hairpin_start(paths, weights, min_identity, max_unitigs, **kw):  # trim.rs:320-326
    return _trim_paths(TRIM_HAIRPIN_START, paths, weights, min_identity, max_unitigs, **kw)


def trim_path_hairpin_end(paths, weights, min_identity, max_unitigs, **kw):    # trim.rs:299-317
    return _trim_paths(TRIM_HAIRPIN_END, paths, weights, min_identity, max_unitigs, **kw)


def trim(cluster_dir, min_identity=0.75, max_unitigs=5000, mad=5.0, threads=8, device=0, verbose=False, lib=None):
    """trim.rs:36-53: reads <cluster_dir>/1_untrimmed.gfa, writes 2_trimmed.gfa and 2_trimmed.yaml."""
    lib = lib or load_library()
    _raise_unless_ok(lib, lib.ac_trim_dir(os.fsencode(cluster_dir), float(min_identity), max_unitigs, float(mad), threads, device, 1 if verbose else 0))


VERBOSE_REPORT, VERBOSE_BANNER = 1, 2


def _dir_array(cluster_dirs):
    names = [os.fsencode(d) for d in cluster_dirs]
    return (C.c_char_p * max(1, len(names)))(*names), len(names)


def trim_dirs(cluster_dirs, min_identity=0.75, max_unitigs=5000, mad=5.0, threads=8, device=0, verbose=False, lib=None):
    """trim() for several cluster directories in one call, every round's alignments of all clusters in one device call.  verbose: True
    for the reports, or VERBOSE_REPORT | VERBOSE_BANNER.  -> the batch info dict: clusters, launches, jobs, cells, buffer_bytes,
    kernel_ms."""
    lib = lib or load_library()
    dirs, n = _dir_array(cluster_dirs)
    info = AcBatchInfo()
    _raise_unless_ok(lib, lib.ac_trim_dirs(dirs, n, float(min_identity), max_unitigs, float(mad), threads, device, int(verbose), C.byref(info)))
    return info.as_dict()


def upgma(matrix, ids, lib=None, device=0, handle=None):
    """UPGMA (cluster.rs:395-480) on the GPU: matrix is a symmetric n x n distance matrix (nested lists or an array) of the clusters `ids`
    (strictly ascending).  -> ([(node, left, right, node distance)] in merge order, kernel milliseconds)."""
    import numpy as np
    lib = lib or load_library()
    h = handle or _Handle(lib, 51, device)
    m = np.ascontiguousarray(np.asarray(matrix, dtype=np.float64))
    n = len(ids)
    assert m.shape == (n, n)
    k = max(1, n - 1)
    node, left, right = (C.c_uint32 * k)(), (C.c_uint32 * k)(), (C.c_uint32 * k)()
    dist = (C.c_double * k)()
    h.check(lib.ac_upgma(h.ptr, m.ctypes.data_as(C.POINTER(C.c_double)), n, (C.c_uint32 * max(1, n))(*ids), node, left, right, dist))
    ms = C.c_float()
    h.check(lib.ac_cluster_stats(h.ptr, None, None, None, None, C.byref(ms), None))
    return [(node[x], left[x], right[x], dist[x]) for x in range(n - 1)], ms.value


def cluster(autocycler_dir, cutoff=0.2, min_assemblies=None, max_contigs=25, manual=None, device=0, verbose=False, lib=None):
    """cluster.rs:30-64: reads <autocycler_dir>/input_assemblies.gfa and replaces <autocycler_dir>/clustering.  manual: "1,2,3"."""
    lib = lib or load_library()
    _raise_unless_ok(lib, lib.ac_cluster_dir(os.fsencode(autocycler_dir), float(cutoff), -1 if min_assemblies is None else int(min_assemblies), max_contigs,
                                             manual.encode() if manual is not None else None, device, 1 if verbose else 0))


def bridge_best_paths(groups, weights, lib=None, device=0, handle=None):
    """Bridge::new (resolve.rs:430-462) for every group of trimmed paths (lists of signed unitig numbers, start and end removed), with the
    distances on the GPU; weights: {unitig: length} or a list indexed by unitig number.  -> ([[u32 total per path]], [best path])"""
    lib = lib or load_library()
    h = handle or _Handle(lib, 51, device)
    w = _weight_list(weights)
    paths = [p for g in groups for p in g]
    flat = [u for p in paths for u in p]
    off, goff = [0], [0]
    for p in paths:
        off.append(off[-1] + len(p))
    for g in groups:
        goff.append(goff[-1] + len(g))
    n, G = len(paths), len(groups)
    totals = (C.c_uint32 * max(1, n))()
    best = (C.c_int32 * max(1, len(flat)))()
    best_off = (C.c_uint64 * (G + 1))()
    h.check(lib.ac_bridge_best_paths(h.ptr, (C.c_int32 * max(1, len(flat)))(*flat), (C.c_uint64 * (n + 1))(*off), n, (C.c_uint64 * (G + 1))(*goff), G,
                                     (C.c_uint32 * max(1, len(w)))(*w), len(w), totals, best, best_off))
    return ([list(totals[goff[g]:goff[g + 1]]) for g in range(G)], [list(best[best_off[g]:best_off[g + 1]]) for g in range(G)])


def resolve(cluster_dir, verbose=False, device=0, lib=None):
    """resolve.rs:31-69: reads <cluster_dir>/2_trimmed.gfa, writes 3_bridged.gfa, 4_merged.gfa and 5_final.gfa."""
    lib = lib or load_library()
    _raise_unless_ok(lib, lib.ac_resolve_dir(os.fsencode(cluster_dir), 1 if verbose else 0, device))


def resolve_dirs(cluster_dirs, verbose=False, device=0, lib=None):
    """resolve() for several cluster directories in one call, all their bridges' distances in one device call.  verbose as for
    trim_dirs.  -> the batch info dict."""
    lib = lib or load_library()
    dirs, n = _dir_array(cluster_dirs)
    info = AcBatchInfo()
    _raise_unless_ok(lib, lib.ac_resolve_dirs(dirs, n, int(verbose), device, C.byref(info)))
    return info.as_dict()


def combine(autocycler_dir, in_gfas, verbose=False, lib=None):
    """combine.rs:25-49: writes <autocycler_dir>/consensus_assembly.gfa, .fasta and .yaml from the GFAs in order."""
    lib = lib or load_library()
    names = [os.fsencode(g) for g in in_gfas]
    _raise_unless_ok(lib, lib.ac_combine_dir(os.fsencode(autocycler_dir), (C.c_char_p * max(1, len(names)))(*names), len(names), 1 if verbose else 0))


def _font_arg(font):
    return None if font is None else os.fsencode(font)


def dotplot_rgb(seqs, res=2000, kmer=32, font=None, device=0, lib=None):
    """create_dotplot (dotplot.rs:179-221) without the file.  seqs: [(filename, name, bytes)], in box order.  font: a TrueType file for
    the labels, "" for none, None for the first standard DejaVuSans.ttf found.  -> ((res, res, 3) uint8 array, info dict: windows,
    groups, dots, host_windows, bp_per_pixel, text_height, kernel_ms)."""
    import numpy as np
    lib = lib or load_library()
    n = len(seqs)
    data = [bytes(s) if not isinstance(s, str) else s.encode() for _, _, s in seqs]
    img = np.empty((res, res, 3), dtype=np.uint8) if 500 <= res <= 10000 else np.empty((1, 1, 3), dtype=np.uint8)
    info = AcDotplotInfo()
    _raise_unless_ok(lib, lib.ac_dotplot_rgb((C.c_char_p * max(1, n))(*data), (C.c_uint64 * max(1, n))(*[len(d) for d in data]),
                                             (C.c_char_p * max(1, n))(*[f.encode() for f, _, _ in seqs]), (C.c_char_p * max(1, n))(*[m.encode() for _, m, _ in seqs]),
                                             n, res, kmer, _font_arg(font), device, img.ctypes.data, C.byref(info)))
    return img, info.as_dict()


def dotplot(input, out_png, res=2000, kmer=32, font=None, device=0, verbose=False, lib=None):
    """dotplot.rs:44-52: input is a directory of assemblies, a FASTA file or an Autocycler GFA; writes out_png.  font as for
    dotplot_rgb.  -> the info dict."""
    lib = lib or load_library()
    info = AcDotplotInfo()
    _raise_unless_ok(lib, lib.ac_dotplot_dir(os.fsencode(input), os.fsencode(out_png), res, kmer, _font_arg(font), device, 1 if verbose else 0, C.byref(info)))
    return info.as_dict()


def png_write(path, rgb, lib=None):
    """An (h, w, 3) uint8 array as an RGB PNG (the encoder `dotplot` uses)."""
    import numpy as np
    lib = lib or load_library()
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    _raise_unless_ok(lib, lib.ac_png_write(os.fsencode(path), rgb.ctypes.data, rgb.shape[1], rgb.shape[0]))


def _host_text(lib, fn, *args):
    """A host-only two-call getter fn(*args, out, cap, length): the length, then the text."""
    n = C.c_uint64()
    _raise_unless_ok(lib, fn(*args, None, 0, C.byref(n)))
    buf = C.create_string_buffer(max(1, n.value))
    _raise_unless_ok(lib, fn(*args, buf, n.value, C.byref(n)))
    return buf.raw[:n.value].decode()


def _depth_arg(min_depth):
    return None if min_depth is None else C.byref(C.c_double(min_depth))


def clean(in_gfa, out_gfa, remove=None, duplicate=None, min_depth=None, verbose=False, lib=None):
    """clean.rs:23-45: remove and duplicate are the CLI's comma-separated tig lists (or None); writes out_gfa.  Host only."""
    lib = lib or load_library()
    _raise_unless_ok(lib, lib.ac_clean_gfa(os.fsencode(in_gfa), os.fsencode(out_gfa), None if remove is None else remove.encode(),
                                           None if duplicate is None else duplicate.encode(), _depth_arg(min_depth), 1 if verbose else 0))


def clean_text(gfa_text, remove=(), duplicate=(), min_depth=None, merge=True, lib=None):
    """clean.rs:26-45 on a GFA text -> the cleaned GFA text.  merge=False stops before merge_linear_paths and renumbering."""
    lib = lib or load_library()
    data = gfa_text.encode() if isinstance(gfa_text, str) else bytes(gfa_text)
    rm, dup = (C.c_uint32 * max(1, len(remove)))(*remove), (C.c_uint32 * max(1, len(duplicate)))(*duplicate)
    return _host_text(lib, lib.ac_clean_text, data, len(data), rm, len(remove), dup, len(duplicate), _depth_arg(min_depth), 1 if merge else 0)


def gfa2fasta(in_gfa, out_fasta, verbose=False, lib=None):
    """gfa2fasta.rs:23-29: writes out_fasta.  Host only."""
    lib = lib or load_library()
    _raise_unless_ok(lib, lib.ac_gfa_to_fasta(os.fsencode(in_gfa), os.fsencode(out_fasta), 1 if verbose else 0))


def gfa_fasta_text(gfa_text, lib=None):
    """save_graph_to_fasta (gfa2fasta.rs:55-82) of a GFA text -> the FASTA text."""
    lib = lib or load_library()
    data = gfa_text.encode() if isinstance(gfa_text, str) else bytes(gfa_text)
    return _host_text(lib, lib.ac_gfa_fasta_text, data, len(data))


def table(autocycler_dir=None, name="", fields=None, sigfigs=3, verbose=False, lib=None):
    """table.rs:24-32 -> the line `autocycler table` prints, newline included: the header without autocycler_dir, else the values."""
    lib = lib or load_library()
    return _host_text(lib, lib.ac_table_text, None if autocycler_dir is None else os.fsencode(autocycler_dir), name.encode(),
                      None if fields is None else fields.encode(), sigfigs, 1 if verbose else 0)


def subsample(reads, out_dir, genome_size, count=4, min_read_depth=25.0, seed=0, device=0, verbose=False, lib=None):
    """`autocycler subsample` (subsample.rs:29-43): sample_01.fastq .. and subsample.yaml under out_dir; returns the info dict."""
    lib = lib or load_library()
    info = AcSubsampleInfo()
    _raise_unless_ok(lib, lib.ac_subsample_dir(os.fsencode(reads), os.fsencode(out_dir), str(genome_size).encode(), count, float(min_read_depth),
                                               seed, device, 1 if verbose else 0, C.byref(info)))
    return info.as_dict()


def genome_size(text, lib=None):   # subsample.rs:83-101
    lib = lib or load_library()
    out = C.c_uint64()
    _raise_unless_ok(lib, lib.ac_genome_size(text.encode(), C.byref(out)))
    return out.value


def subsample_words(seed, n, rounds=12, lib=None):
    """The first n u32 words of StdRng::seed_from_u64(seed) (ChaCha12), or of its 20-round form."""
    lib = lib or load_library()
    out = (C.c_uint32 * max(1, n))()
    _raise_unless_ok(lib, lib.ac_subsample_words(seed, rounds, out, n))
    return list(out)[:n]


def subsample_shuffle(n, seed, lib=None):
    """(0..n).shuffle(&mut StdRng::seed_from_u64(seed)) as a list."""
    lib = lib or load_library()
    out = (C.c_uint32 * max(1, n))()
    _raise_unless_ok(lib, lib.ac_subsample_shuffle(n, seed, out))
    return list(out)[:n]


def genome_size_estimate(reads, k=21, device=0, dir=None, verbose=False, lib=None):
    """`autocycler helper genome_size`: the genome size from the reads' k-mer depth spectrum (DESIGN.md §18; not the reference's Raven
    assembly length).  Returns the info dict, with "histogram": the AC_GENOME_SIZE_BINS bins as a list."""
    lib = lib or load_library()
    info = AcGenomeSizeInfo()
    hist = (C.c_uint64 * GENOME_SIZE_BINS)()
    _raise_unless_ok(lib, lib.ac_genome_size_estimate(os.fsencode(reads), k, device, None if dir is None else os.fsencode(dir),
                                                      1 if verbose else 0, hist, C.byref(info)))
    out = info.as_dict()
    out["histogram"] = list(hist)
    return out


def genome_size_from_histogram(hist, windows, lib=None):
    """The rule alone (host only) on a histogram of up to AC_GENOME_SIZE_BINS bins (zero-padded) and its window count -> the info dict."""
    lib = lib or load_library()
    if len(hist) > GENOME_SIZE_BINS:
        raise ValueError(f"at most {GENOME_SIZE_BINS} bins")
    h = (C.c_uint64 * GENOME_SIZE_BINS)(*[int(x) for x in hist])
    info = AcGenomeSizeInfo()
    _raise_unless_ok(lib, lib.ac_genome_size_from_histogram(h, windows, C.byref(info)))
    return info.as_dict()


def _fasta_records(path):
    """The number of records of a FASTA file (gzipped or not): its lines that start with '>'."""
    import gzip
    with open(path, "rb") as f:
        data = f.read()
    if data[:2] == b"\x1f\x8b":
        data = gzip.decompress(data)
    return sum(1 for line in data.split(b"\n") if line.startswith(b">"))


def depth(assembly, out_fasta, reads=None, source="reads", k=21, min_depth_abs=None, min_depth_rel=None, tsv=None, device=0, verbose=False,
          lib=None):
    """`autocycler depth` (DESIGN.md §19): each contig's read depth from the reads' k-mers, counted on the GPU (not in the reference), then
    the reference's helper depth filter; source="header" is that filter alone on the headers' depths.  Returns the info dict, with
    "depths" (per contig, None without a depth) and "unique" (per contig, its unique k-mers)."""
    lib = lib or load_library()
    if source not in ("reads", "header"):
        raise ValueError("source must be 'reads' or 'header'")
    cap = _fasta_records(assembly) if os.path.isfile(assembly) else 0
    depths = (C.c_double * max(1, cap))()
    unique = (C.c_uint64 * max(1, cap))()
    info = AcDepthInfo()
    _raise_unless_ok(lib, lib.ac_depth_fasta(os.fsencode(assembly), None if reads is None else os.fsencode(reads), os.fsencode(out_fasta),
                                             None if tsv is None else os.fsencode(tsv), 1 if source == "header" else 0, k,
                                             _depth_arg(min_depth_abs), _depth_arg(min_depth_rel), device, 1 if verbose else 0, depths,
                                             unique, cap, C.byref(info)))
    out = info.as_dict()
    n = min(cap, out["contigs"])
    out["depths"] = [None if d != d else d for d in list(depths)[:n]]
    out["unique"] = list(unique)[:n]
    return out


def depth_filter_text(fasta_text, min_depth_abs=None, min_depth_rel=None, lib=None):
    """helper.rs:889-921 on a FASTA text -> what the file holds afterwards ("" when nothing is kept).  Host only."""
    lib = lib or load_library()
    data = fasta_text.encode() if isinstance(fasta_text, str) else fasta_text
    return _host_text(lib, lib.ac_depth_filter_text, data, len(data), _depth_arg(min_depth_abs), _depth_arg(min_depth_rel))


def depth_from_header(header, lib=None):
    """helper.rs:923-931: the depth a FASTA header carries, or None.  Host only."""
    lib = lib or load_library()
    d = C.c_double()
    rc = lib.ac_depth_from_header(header.encode(), C.byref(d))
    if rc == -6:
        return None
    _raise_unless_ok(lib, rc)
    return d.value


def qv(reads, assemblies, out_dir, k=21, min_count=None, device=0, verbose=False, lib=None):
    """`autocycler qv` (DESIGN.md §20): each assembly's k-mer QV and completeness against the reads, counted on the GPU (not in the
    reference).  assemblies: FASTA files or directories (expanded as find_all_assemblies does).  Returns the info dict (t is "min_count", S
    "solid_kmers", the stage timings in ms) with "assemblies": per assembly a dict of path, kmers, unsupported, solid_found and qv (None for
    an empty field, float("inf") for inf), and "contigs": per contig a dict of assembly, contig, length, kmers, unsupported and qv, both
    read back from the qv.tsv and contig_qv.tsv the call wrote."""
    lib = lib or load_library()
    paths = [assemblies] if isinstance(assemblies, (str, bytes, os.PathLike)) else list(assemblies)
    cap = sum(len(os.listdir(p)) if os.path.isdir(p) else 1 for p in paths)
    arr = (C.c_char_p * max(1, len(paths)))(*[os.fsencode(p) for p in paths])
    kmers, unsupported, found = ((C.c_uint64 * max(1, cap))() for _ in range(3))
    info = AcQvInfo()
    t = None if min_count is None else C.byref(C.c_uint32(min_count))
    _raise_unless_ok(lib, lib.ac_qv_dir(os.fsencode(reads), arr, len(paths), os.fsencode(out_dir), k, t, device, 1 if verbose else 0, kmers,
                                        unsupported, found, cap, C.byref(info)))
    out = info.as_dict()

    def rows(name):
        with open(os.path.join(out_dir, name)) as f:
            lines = f.read().splitlines()
        head = lines[0].split("\t")
        return [dict(zip(head, line.split("\t"))) for line in lines[1:]]

    def qv_value(text):
        return None if text == "" else float(text)

    n = min(cap, out["assemblies"])
    out["assemblies"] = [{"path": r["assembly"], "kmers": kmers[i], "unsupported": unsupported[i], "solid_found": found[i],
                          "qv": qv_value(r["qv"]), "completeness": qv_value(r["completeness"])} for i, r in enumerate(rows("qv.tsv")[:n])]
    out["contigs"] = [{"assembly": r["assembly"], "contig": r["contig"], "length": int(r["length"]), "kmers": int(r["kmers"]),
                       "unsupported": int(r["unsupported"]), "qv": qv_value(r["qv"])} for r in rows("contig_qv.tsv")]
    return out


def unassembled(reads, assemblies, out_dir, k=21, min_count=None, min_solid=100, min_fraction=0.5, device=0, verbose=False, lib=None):
    """`autocycler unassembled` (DESIGN.md §21): the reads the assembly does not explain, and the depth of the sequence it misses,
    counted on the GPU (not in the reference).  assemblies: FASTA files or directories (expanded as find_all_assemblies does); together
    they are the assembly.  Returns the info dict (t is "min_count"; absent_median, peak and absent_copy_ratio are None where summary.tsv
    leaves them empty; the stage timings in ms) with "selected": per selected read a dict of read, length, solid_kmers and absent_kmers,
    read back from the unassembled.tsv the call wrote."""
    lib = lib or load_library()
    paths = [assemblies] if isinstance(assemblies, (str, bytes, os.PathLike)) else list(assemblies)
    arr = (C.c_char_p * max(1, len(paths)))(*[os.fsencode(p) for p in paths])
    info = AcUnassembledInfo()
    t = None if min_count is None else C.byref(C.c_uint32(min_count))
    _raise_unless_ok(lib, lib.ac_unassembled_dir(os.fsencode(reads), arr, len(paths), os.fsencode(out_dir), k, t, min_solid, min_fraction, device,
                                                 1 if verbose else 0, C.byref(info)))
    out = info.as_dict()
    for name in ("absent_median", "peak", "absent_copy_ratio"):
        if out[name] != out[name]:
            out[name] = None
    with open(os.path.join(out_dir, "unassembled.tsv")) as f:
        lines = f.read().splitlines()
    out["selected"] = [{"read": r[0], "length": int(r[1]), "solid_kmers": int(r[2]), "absent_kmers": int(r[3])}
                       for r in (line.split("\t") for line in lines[1:])]
    return out


def polish(reads, assembly, out_dir, k=21, min_count=None, max_indel=3, rounds=3, device=0, verbose=False, lib=None):
    """`autocycler polish` (DESIGN.md §22): the consensus corrected where the reads' k-mers do not support it, with candidate edits
    scored on the GPU (not in the reference).  Returns the info dict (t is "min_count", the stage timings in ms) with "qv_before" and
    "qv_after" (None for an empty field, float("inf") for inf) and "applied": per applied edit a dict of round, contig, position, ref, alt
    and score, both read back from the summary.tsv and edits.tsv the call wrote."""
    lib = lib or load_library()
    info = AcPolishInfo()
    t = None if min_count is None else C.byref(C.c_uint32(min_count))
    _raise_unless_ok(lib, lib.ac_polish_fasta(os.fsencode(reads), os.fsencode(assembly), os.fsencode(out_dir), k, t, max_indel, rounds, device,
                                              1 if verbose else 0, C.byref(info)))
    out = info.as_dict()
    with open(os.path.join(out_dir, "summary.tsv")) as f:
        head, row = (line.split("\t") for line in f.read().splitlines())
    summary = dict(zip(head, row))
    for name in ("qv_before", "qv_after"):
        out[name] = None if summary[name] == "" else float(summary[name])
    with open(os.path.join(out_dir, "edits.tsv")) as f:
        lines = f.read().splitlines()
    out["applied"] = [{"round": int(r[0]), "contig": r[1], "position": int(r[2]), "ref": r[3], "alt": r[4], "score": int(r[5])}
                    for r in (line.split("\t") for line in lines[1:])]
    return out


def variants(reads, assembly, out_dir, k=21, min_count=None, max_indel=1, min_fraction=0.1, device=0, verbose=False, lib=None):
    """`autocycler variants` (DESIGN.md §23): the alleles the reads carry beside the consensus, with every position's alternatives
    screened on the GPU (not in the reference).  Returns the info dict (t is "min_count", the stage timings in ms) with "rows": per row of
    the variants.vcf the call wrote a dict of contig, pos, ref, alt, af, ak, rk and pk."""
    lib = lib or load_library()
    info = AcVariantsInfo()
    t = None if min_count is None else C.byref(C.c_uint32(min_count))
    _raise_unless_ok(lib, lib.ac_variants_fasta(os.fsencode(reads), os.fsencode(assembly), os.fsencode(out_dir), k, t, max_indel, min_fraction,
                                                device, 1 if verbose else 0, C.byref(info)))
    out = info.as_dict()
    rows = []
    with open(os.path.join(out_dir, "variants.vcf")) as f:
        for line in f:
            if line.startswith("#"):
                continue
            c = line.rstrip("\n").split("\t")
            tags = dict(x.split("=") for x in c[7].split(";"))
            rows.append({"contig": c[0], "pos": int(c[1]), "ref": c[3], "alt": c[4], "af": float(tags["AF"]), "ak": int(tags["AK"]),
                         "rk": int(tags["RK"]), "pk": int(tags["PK"])})
    out["rows"] = rows
    return out
