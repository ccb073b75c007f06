"""CPU oracle of `autocycler cluster` (rrwick/Autocycler v0.6.1, cluster.rs) — test infrastructure only.

A restatement of cluster.rs:30-912 in Python on the text of input_assemblies.gfa.  The distances are computed from the GFA itself
(cluster.rs:132-151, with a_len the u32 sum the reference converts).  `upgma` keeps the clusters' distance sums over member pairs
(T(A u B, C) = T(A, C) + T(B, C), mean = T / (|A| |C|)), the averaging the product documents in DESIGN.md §12; `upgma_reference` is a
literal port of the reference's loop, which averages over every member pair, to check that restatement.  Where the reference's order is a
HashMap's, the product's fixed order is used: the balance score sums clusters in ascending number and a contained cluster names the
smallest passed cluster that contains it.  The per-cluster graphs go through the C++ oracle's merge_linear_paths
(oracle_lib.gfa_merge_linear_paths, renumber=False)."""
import math
from decimal import Decimal

import numpy as np

import oracle_lib


# ---- number formats ---------------------------------------------------------------------------------------------------------------

def _digits(v):
    """shortest round-trip digits of v > 0 and the position of the decimal point: v = 0.d1d2... x 10^point"""
    t = Decimal(repr(float(v))).normalize().as_tuple()
    d = "".join(map(str, t.digits))
    return d, len(d) + t.exponent


def rust_display(v):   # Rust's `{}` for f64: never an exponent, no trailing .0
    if math.isnan(v):
        return "NaN"
    if math.isinf(v):
        return "inf" if v > 0 else "-inf"
    sign = "-" if math.copysign(1.0, v) < 0 else ""
    if v == 0:
        return sign + "0"
    d, p = _digits(abs(v))
    if p <= 0:
        return sign + "0." + "0" * -p + d
    if p >= len(d):
        return sign + d + "0" * (p - len(d))
    return sign + d[:p] + "." + d[p:]


def yaml_float(v):     # serde_yaml 0.9 (ryu 1.0): derived from ryu's layout rules, not compared against the crate
    if math.isnan(v):
        return ".nan"
    if math.isinf(v):
        return ".inf" if v > 0 else "-.inf"
    sign = "-" if math.copysign(1.0, v) < 0 else ""
    if v == 0:
        return sign + "0.0"
    d, kk = _digits(abs(v))
    k = kk - len(d)
    if k >= 0 and kk <= 16:
        return sign + d + "0" * k + ".0"
    if 0 < kk <= 16:
        return sign + d[:kk] + "." + d[kk:]
    if -5 < kk <= 0:
        return sign + "0." + "0" * -kk + d
    if len(d) == 1:
        return f"{sign}{d}e{kk - 1}"
    return f"{sign}{d[0]}.{d[1:]}e{kk - 1}"


def format_float(v):   # misc.rs:363-370
    s = f"{v:.6f}"
    if "." not in s:
        return s
    return s.rstrip("0").rstrip(".")


# ---- sequences --------------------------------------------------------------------------------------------------------------------

class Seq:
    def __init__(self, id, path, length, filename, header):
        self.id, self.path, self.length, self.filename, self.header = id, path, length, filename, header
        self.cluster = 0

    def _weight(self, key):   # sequence.rs:97-109
        for tok in self.header.lower().split():
            if tok.startswith(key):
                v = tok[len(key):]
                w = v[1:] if v.startswith("+") else v
                if w and w.isdigit() and w.isascii():
                    return int(w)
        return 1

    def cluster_weight(self):
        return self._weight("autocycler_cluster_weight=")

    def consensus_weight(self):
        return self._weight("autocycler_consensus_weight=")

    def trusted(self):
        return "autocycler_trusted" in self.header.lower()

    def contig_name(self):
        return self.header.split(" ")[0]

    def newick(self):
        return f"{self.id}__{self.filename}__{self.contig_name()}__{self.length}_bp"


def parse_gfa(text):
    lines = [ln[:-1] if ln.endswith("\r") else ln for ln in text.split("\n") if ln]
    lengths = {}
    seqs = []
    for ln in lines:
        p = ln.split("\t")
        if p[0] == "S":
            lengths[int(p[1])] = len(p[2])
        elif p[0] == "P":
            tags = {x[:5]: x[5:] for x in p[3:]}
            path = [int(s[:-1]) for s in p[2].split(",")] if p[2] else []
            seqs.append(Seq(int(p[1]), path, int(tags["LN:i:"]), tags["FN:Z:"], tags["HD:Z:"]))
    return lengths, seqs


def distances(lengths, seqs):   # cluster.rs:132-151 -> asymmetric matrix in sequence order
    sets = [set(s.path) for s in seqs]
    n = len(seqs)
    d = np.zeros((n, n))
    for a in range(n):
        a_len = float(sum(lengths[u] for u in sets[a]) & 0xFFFFFFFF)
        for b in range(n):
            d[a, b] = 1.0 - (float(sum(lengths[u] for u in sets[a] & sets[b])) / a_len)
    return d


def symmetric(d):   # cluster.rs:177-192
    return np.maximum(d, d.T)


# ---- UPGMA ------------------------------------------------------------------------------------------------------------------------

def upgma(sym, ids):
    """UPGMA with distance sums: -> [(node, left, right, node distance)].  The least (distance, a, b) over live pairs a < b (ascending id
    order) merges; b joins a (new_id = a.min(b)); nodes are numbered from max(ids) + 1."""
    n = len(ids)
    assert list(ids) == sorted(set(ids))
    T = np.array(sym, dtype=np.float64, copy=True)
    D = np.full((n, n), np.inf)
    iu = np.triu_indices(n, 1)
    D[iu] = T[iu]
    cnt = np.ones(n, dtype=np.int64)
    node = list(ids)
    alive = np.ones(n, dtype=bool)
    merges = []
    nxt = max(ids) if ids else 0
    for _ in range(n - 1):
        x = int(np.argmin(D))                 # row-major: the first least pair in (a, b) order
        a, b = divmod(x, n)
        dist = D[a, b]
        nxt += 1
        merges.append((nxt, node[a], node[b], dist / 2.0))
        node[a] = nxt
        alive[b] = False
        D[b, :] = np.inf
        D[:, b] = np.inf
        cnt[a] += cnt[b]
        T[a, :] = T[a, :] + T[b, :]
        T[:, a] = T[a, :]
        js = np.nonzero(alive)[0]
        js = js[js != a]
        vals = T[a, js] / (cnt[a] * cnt[js]).astype(np.float64)
        lo, hi = js < a, js > a
        D[js[lo], a] = vals[lo]
        D[a, js[hi]] = vals[hi]
    return merges


def upgma_reference(sym, ids):
    """cluster.rs:395-480 as written: every merge re-averages the original distances over all member pairs."""
    dist = {(ids[i], ids[j]): float(sym[i][j]) for i in range(len(ids)) for j in range(len(ids))}
    clusters = {i: {i} for i in ids}
    cd = dict(dist)
    nxt = max(ids)
    merges = []
    while len(clusters) > 1:
        keys = sorted({k for pair in cd for k in pair})
        best, pair = math.inf, (0, 0)
        for x, a in enumerate(keys):
            for b in keys[x + 1:]:
                v = cd.get((a, b), cd.get((b, a)))
                if v is not None and v < best:
                    best, pair = v, (a, b)
        a, b = pair
        ca, cb = clusters.pop(a), clusters.pop(b)
        new_id = min(a, b)
        clusters[new_id] = ca | cb
        nxt += 1
        merges.append((nxt, a, b, best / 2.0))
        nd = {k: v for k, v in cd.items() if k[0] in clusters and k[1] in clusters}
        for o in clusters:
            if o != new_id:
                s, c = 0.0, 0
                for i1 in clusters[new_id]:
                    for i2 in clusters[o]:
                        s += dist[(i1, i2)]
                        c += 1
                nd[(new_id, o)] = nd[(o, new_id)] = s / c
        cd = nd
    # the reference's children are nodes; map the cluster ids of each merge to the node that cluster last became
    last = {i: i for i in ids}
    out = []
    for node, a, b, d in merges:
        out.append((node, last[a], last[b], d))
        last[min(a, b)] = node
    return out


# ---- the tree ---------------------------------------------------------------------------------------------------------------------

class Tree:
    def __init__(self, ids, merges):
        self.left, self.right, self.dist = {}, {}, {i: 0.0 for i in ids}
        self.root = ids[0] if ids else 0
        for node, l, r, d in merges:
            self.left[node], self.right[node], self.dist[node] = l, r, d
            self.root = node

    def tip(self, u):
        return u not in self.left

    def normalise(self):   # cluster.rs:483-494
        if self.dist[self.root] > 0.5:
            f = 0.5 / self.dist[self.root]
            for u in self.dist:
                self.dist[u] *= f

    def tips(self, u):
        return [u] if self.tip(u) else self.tips(self.left[u]) + self.tips(self.right[u])

    def newick(self, u, by_id):   # cluster.rs:381-392
        if self.tip(u):
            return by_id[u].newick()
        l, r = self.left[u], self.right[u]
        return (f"({self.newick(l, by_id)}:{rust_display(self.dist[u] - self.dist[l])},"
                f"{self.newick(r, by_id)}:{rust_display(self.dist[u] - self.dist[r])}){u}")

    def find(self, u):   # find_node (:337-347)
        return u if u in self.dist else None

    def max_pairwise_distance(self, u):   # :208-217
        return self.dist[u] * 2.0 if u in self.dist else -1.0

    def check_complete_coverage(self, clusters):   # :297-309
        seen = [t for c in clusters for t in self.tips(c)]
        if len(seen) != len(set(seen)):
            raise ValueError("overlap detected")
        if set(seen) != set(self.tips(self.root)):
            raise ValueError("incomplete coverage")

    def has_manual(self, u, manual):
        return u in manual or (not self.tip(u) and (self.has_manual(self.left[u], manual) or self.has_manual(self.right[u], manual)))

    def collect(self, u, cutoff, manual, out):   # cluster.rs:239-247
        if u in manual or (self.dist[u] <= cutoff and not self.has_manual(u, manual)):
            out.append(u)
        elif not self.tip(u):
            self.collect(self.left[u], cutoff, manual, out)
            self.collect(self.right[u], cutoff, manual, out)

    def check_consistency(self, u, manual):   # cluster.rs:260-271
        if not self.tip(u):
            if u in manual and (self.has_manual(self.left[u], manual) or self.has_manual(self.right[u], manual)):
                raise ValueError("manual clusters cannot be nested")
            self.check_consistency(self.left[u], manual)
            self.check_consistency(self.right[u], manual)

    def splits(self, clusters):   # cluster.rs:311-335
        res = []
        for c in clusters:
            if not self.tip(c):
                res.append(sorted([o for o in clusters if o != c] + [self.left[c], self.right[c]]))
        return sorted(res)


def _median(v):
    if not v:
        return 0
    v = sorted(v)
    n = len(v)
    return (v[n // 2 - 1] + v[n // 2]) // 2 if n % 2 == 0 else v[n // 2]


def _mad(v):
    if not v:
        return 0
    m = _median(v)
    return _median([abs(x - m) for x in v])


def cluster_assembly_count(seqs, c):   # cluster.rs:573-585
    w = {}
    for s in seqs:
        if s.cluster == c:
            w[s.filename] = max(w.get(s.filename, 0), s.cluster_weight())
    return sum(w.values())


def set_min_assemblies(option, seqs):   # cluster.rs:645-661
    if option is not None:
        return option
    files = {s.filename for s in seqs}
    return 1 if len(files) == 1 else max(2, (len(files) + 2) // 4)


def reorder_clusters(seqs):   # cluster.rs:881-902 -> {old: new}
    C = max(s.cluster for s in seqs)
    med = {c: _median([s.length for s in seqs if s.cluster == c]) for c in range(1, C + 1)}
    new = {old: k + 1 for k, old in enumerate(sorted(med, key=lambda c: (-med[c], c)))}
    for s in seqs:
        if s.cluster >= 1:
            s.cluster = new[s.cluster]
    return new


def parse_manual_clusters(text):   # cluster.rs:664-671
    if text is None:
        return []
    out = []
    for s in text.replace(" ", "").split(","):
        t = s[1:] if s.startswith("+") else s
        if not (t and t.isascii() and t.isdigit() and int(t) <= 0xFFFF):
            raise ValueError(f"failed to parse '{s}' as a node number")
        out.append(int(t))
    return sorted(out)


def qc_clusters(tree, seqs, asym, nodes, manual, cutoff, min_assemblies):   # cluster.rs:511-570 -> [(reasons, dist)] per cluster
    index = {s.id: i for i, s in enumerate(seqs)}
    qc = []
    for n in nodes:
        if n not in tree.dist:
            raise ValueError(f"clustering tree does not contain a node with id {n}")
        for t in tree.tips(n):
            seqs[index[t]].cluster = len(qc) + 1
        qc.append(([] if not manual or n in manual else ["not included in manual clusters"], tree.dist[n] * 2.0))
    C = len(qc)
    new = reorder_clusters(seqs)
    qc = [qc[old - 1] for old in sorted(new, key=new.get)]
    if manual:
        return qc
    for c in range(1, C + 1):
        members = [s for s in seqs if s.cluster == c]
        if cluster_assembly_count(seqs, c) < min_assemblies and not any(s.trusted() for s in members):
            qc[c - 1][0].append("present in too few assemblies")
    for c in range(1, C + 1):
        ia = [i for i, s in enumerate(seqs) if s.cluster == c]
        for p in range(1, C + 1):
            if p == c or qc[p - 1][0]:
                continue
            ib = [i for i, s in enumerate(seqs) if s.cluster == p]
            cc = sum(1 for a in ia for b in ib if asym[a, b] < asym[b, a] and asym[a, b] < cutoff)
            if cc / (len(ia) * len(ib)) > 0.5:
                if not any(seqs[i].trusted() for i in ia):
                    qc[c - 1][0].append(f"contained within cluster {p}")
                break
    return qc


def metrics(seqs, qc):   # clustering_metrics + ClusteringMetrics (metrics.rs:123-183)
    m = {"pass_cluster_count": sum(1 for r, _ in qc if not r), "fail_cluster_count": sum(1 for r, _ in qc if r)}
    m["pass_contig_count"] = sum(1 for s in seqs if not qc[s.cluster - 1][0])
    m["fail_contig_count"] = len(seqs) - m["pass_contig_count"]
    total = len(seqs)
    m["pass_contig_fraction"] = m["pass_contig_count"] / total if total else 0.0
    m["fail_contig_fraction"] = m["fail_contig_count"] / total if total else 0.0
    files = {s.filename for s in seqs}
    weighted, tw = 0.0, 0.0
    for c in range(1, len(qc) + 1):
        names = [s.filename for s in seqs if s.cluster == c]
        score = sum(1.0 if names.count(f) == 1 else 0.0 for f in files) / float(len(files))
        weighted += score * float(len(names))
        tw += float(len(names))
    m["cluster_balance_score"] = weighted / tw
    pd = [d for r, d in qc if not r]
    t = 0.0
    for d in pd:
        t += 1.0 - math.sqrt(d)
    m["cluster_tightness_score"] = t / len(pd) if pd else 0.0
    m["overall_clustering_score"] = (m["cluster_balance_score"] + m["cluster_tightness_score"]) / 2.0
    return m


def metrics_yaml(m):
    out = ""
    for k, v in m.items():
        out += f"{k}: {yaml_float(v) if isinstance(v, float) else v}\n"
    return out


def untrimmed_yaml(lengths, dist):   # UntrimmedClusterMetrics (metrics.rs:186-205)
    y = f"untrimmed_cluster_size: {len(lengths)}\n"
    y += "untrimmed_cluster_lengths: []\n" if not lengths else "untrimmed_cluster_lengths:\n" + "".join(f"- {x}\n" for x in lengths)
    return y + f"untrimmed_cluster_median: {_median(lengths) & 0xFFFFFFFF}\nuntrimmed_cluster_mad: {_mad(lengths) & 0xFFFFFFFF}\n" \
               f"untrimmed_cluster_distance: {yaml_float(dist)}\n"


def cluster_gfa(text, seqs, c):   # save_cluster_gfa (cluster.rs:794-806)
    keep_ids = {s.id for s in seqs if s.cluster == c}
    lines = [ln[:-1] if ln.endswith("\r") else ln for ln in text.split("\n") if ln]
    paths = [ln.split("\t") for ln in lines if ln.startswith("P\t") and (not ln.split("\t")[1].isdigit() or int(ln.split("\t")[1]) in keep_ids)]
    depth = {}
    for p in paths:
        for s in (p[2].split(",") if p[2] else []):
            depth[int(s[:-1])] = depth.get(int(s[:-1]), 0) + 1
    out = []
    for ln in lines:
        p = ln.split("\t")
        if p[0] == "S":
            n = int(p[1])
            if depth.get(n, 0) > 0:
                out.append("\t".join(p[:3] + [f"DP:f:{float(depth[n]):.2f}" if x.startswith("DP:f:") else x for x in p[3:]]))
        elif p[0] == "L":
            if depth.get(int(p[1]), 0) > 0 and depth.get(int(p[3]), 0) > 0:
                out.append(ln)
        elif p[0] == "P":
            if p in paths:
                out.append(ln + f"\tCL:i:{c}")
        else:
            out.append(ln)
    return oracle_lib.gfa_merge_linear_paths("\n".join(out) + "\n", use_paths=True, renumber=False)


def cluster(gfa_text, cutoff=0.2, min_assemblies=None, manual=None):
    """cluster.rs:42-59 -> {relative path under clustering/: text}"""
    lengths, seqs = parse_gfa(gfa_text)
    min_assemblies = set_min_assemblies(min_assemblies, seqs)
    manual = sorted(manual or [])
    asym = distances(lengths, seqs)
    order = sorted(range(len(seqs)), key=lambda i: seqs[i].id)
    ids = [seqs[i].id for i in order]
    sym = symmetric(asym)[np.ix_(order, order)]
    tree = Tree(ids, upgma(sym, ids))
    tree.normalise()
    by_id = {s.id: s for s in seqs}
    nw = tree.newick(tree.root, by_id)
    r = tree.dist[tree.root]
    out = {"clustering.newick": f"({nw}:{rust_display(0.5 - r)});\n" if r < 0.5 else f"{nw};\n"}
    if not manual:
        nodes = []
        tree.collect(tree.root, cutoff / 2.0, [], nodes)
        best = sorted(nodes)
        best_score = metrics(seqs, qc_clusters(tree, seqs, asym, best, [], cutoff, min_assemblies))["overall_clustering_score"]
        improved = True
        while improved:
            improved = False
            for alt in tree.splits(best):
                s = metrics(seqs, qc_clusters(tree, seqs, asym, alt, [], cutoff, min_assemblies))["overall_clustering_score"]
                if s > best_score:
                    best, best_score, improved = alt, s, True
        nodes = best
    else:
        tree.check_consistency(tree.root, manual)
        nodes = []
        tree.collect(tree.root, cutoff / 2.0, manual, nodes)
        nodes.sort()
    qc = qc_clusters(tree, seqs, asym, nodes, manual, cutoff, min_assemblies)
    out["pairwise_distances.phylip"] = oracle_lib.pairwise_distances(gfa_text)
    for c in range(1, len(qc) + 1):
        d = f"{'qc_fail' if qc[c - 1][0] else 'qc_pass'}/cluster_{c:03d}"
        out[f"{d}/1_untrimmed.gfa"] = cluster_gfa(gfa_text, seqs, c)
        out[f"{d}/1_untrimmed.yaml"] = untrimmed_yaml([s.length for s in seqs if s.cluster == c], qc[c - 1][1])
    tsv = "node_name\tpassing_clusters\tall_clusters\tsequence_id\tfile_name\tcontig_name\tlength\ttrusted\tcluster_weight\tconsensus_weight\n"
    for s in seqs:
        p = str(s.cluster) if not qc[s.cluster - 1][0] else "none"
        tsv += (f"{s.newick()}\t{p}\t{s.cluster}\t{s.id}\t{s.filename}\t{s.contig_name()}\t{s.length}\t{'true' if s.trusted() else 'false'}\t"
                f"{s.cluster_weight()}\t{s.consensus_weight()}\n")
    out["clustering.tsv"] = tsv
    out["clustering.yaml"] = metrics_yaml(metrics(seqs, qc))
    return out
