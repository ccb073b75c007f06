"""Shared body of the parity tests: run one case through a C-ABI library (the CUDA build on the GPU box, or
the host-emulation build of the same device bodies on CPU) and compare with the oracle."""
import tempfile

import cases
import oracle_lib as o
from autocycler_b200 import api


def run_library(lib, directory, k, positions=False):
    kg, seqs, count = api.load_sequences(directory, k, lib=lib)
    if positions:
        kg2 = api.KmerGraph(k, lib=lib, keep_positions=True)
        kg2.add_sequences(seqs, count)
        kg = kg2
    else:
        kg.upload()
    graph = api.UnitigGraph.from_kmer_graph(kg)
    before = graph.counts()
    seed_state = graph.unitigs(positions=True) if positions else None
    api.simplify_structure(graph)
    after = graph.counts()
    return dict(gfa=graph.gfa_bytes().decode(), before=before, after=after, seqs=seqs, count=count, graph=graph,
                seed_state=seed_state, kg=kg)


def check_fused(kg, expected, st, seqs, k):
    """ac_compress — compress.rs:42-47 as one device pipeline — on the same sequences: the same file, the counts compress prints, and
    a graph (fetched from HBM on first use) that behaves like the one the step-by-step calls built."""
    kg.upload()
    g = api.UnitigGraph.compress(kg)
    c = g.counts()                                         # before anything asks for the graph: the device's own counts
    assert (c.n_kmers, c.n_unitigs, c.n_links, c.total_length, c.length_before_simplify) == \
           (st.n_kmers, st.unitigs_after, st.links_after, st.length_after, st.length_before)
    assert bytes(g.gfa_view()).decode() == expected, "fused build: GFA differs from the oracle"
    assert g.distance_matrix_text() == o.pairwise_distances(expected)
    c = g.counts()                                         # now from the adopted host graph
    assert (c.n_unitigs, c.n_links, c.total_length) == (st.unitigs_after, st.links_after, st.length_after)
    originals = [s.forward_seq[k // 2: len(s.forward_seq) - k // 2] for s in seqs]
    assert [g.reconstruct_original_sequence(i) for i in range(len(originals))] == originals
    api.simplify_structure(g)                              # nothing left to do
    assert g.gfa_bytes().decode() == expected
    api.merge_linear_paths(g, seqs)
    assert g.gfa_bytes().decode() == o.gfa_merge_linear_paths(expected)
    g.renumber_unitigs()
    assert g.gfa_bytes().decode() == o.gfa_merge_linear_paths(expected, renumber=True)
    return g


def check_case(lib, files, k, tmpdir=None):
    with tempfile.TemporaryDirectory(dir=tmpdir) as d:
        cases.write_case(files, d)
        try:
            expected, yaml, st = o.compress_dir(d, k)
        except o.OracleError as e:
            # the reference rejects this input (quit_with_error); the library must reject it too
            try:
                run_library(lib, d, k)
            except api.AutocyclerGpuError:
                return None
            raise AssertionError(f"oracle rejected the input ({e}) but the library accepted it")
        count, oseqs = o.load_sequences(d, k)
        got = run_library(lib, d, k)
        assert [(s.id, s.filename, s.contig_header, s.length, s.forward_seq) for s in got["seqs"]] == oseqs, "load/end-repair differs"
        assert got["count"] == count
        assert got["before"].n_kmers == st.n_kmers
        assert (got["before"].n_unitigs, got["before"].n_links, got["before"].total_length) == \
               (st.unitigs_before, st.links_before, st.length_before)
        assert (got["after"].n_unitigs, got["after"].n_links, got["after"].total_length) == \
               (st.unitigs_after, st.links_after, st.length_after)
        assert got["gfa"] == expected, "GFA differs from the oracle"
        assert got["graph"].distance_matrix_text() == o.pairwise_distances(expected), "distance matrix (cluster.rs:132-176) differs from the oracle"
        originals = [s.forward_seq[k // 2: len(s.forward_seq) - k // 2] for s in got["seqs"]]
        # tests.rs:114-127: every input contig comes back from its path (end repair only ever touches the dots)
        assert [got["graph"].reconstruct_original_sequence(i) for i in range(len(originals))] == originals
        # what every downstream command does next (cluster.rs:804): merge_linear_paths on the loaded graph
        api.merge_linear_paths(got["graph"], got["seqs"])
        got["merged_gfa"] = got["graph"].gfa_bytes().decode()
        assert got["merged_gfa"] == o.gfa_merge_linear_paths(expected), "merged GFA differs from the oracle"
        assert [got["graph"].reconstruct_original_sequence(i) for i in range(len(originals))] == originals
        got["graph"].renumber_unitigs()     # trim.rs:266-268: merge, then renumber
        assert got["graph"].gfa_bytes().decode() == o.gfa_merge_linear_paths(expected, renumber=True), "renumbered merged GFA differs"
        check_fused(got["kg"], expected, st, got["seqs"], k)
        return got


def check_distances(graph, gfa_text):
    """cluster.rs:132-176 on the graph `gfa_text` was saved from: same matrix file as the oracle's restatement writes."""
    assert graph.distance_matrix_text() == o.pairwise_distances(gfa_text)
