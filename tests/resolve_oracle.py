"""CPU oracle of `autocycler resolve` and `autocycler combine` (rrwick/Autocycler v0.6.1, resolve.rs and combine.rs) — test infrastructure
only.

A literal restatement in Python: the ordered P^2 loop of Bridge::new over global_alignment_distance in u32 with wraparound (the reference
ships as a release build, overflow checks off), determine_ambiguity, the quadratic cull loop, and apply_bridges with the link edits of
unitig_graph.rs:795-903 on per-strand lists.  merge_linear_paths + renumber_unitigs + save_gfa go to the C++ oracle
(oracle_lib.gfa_merge_linear_paths), which re-loads the bridged graph from its text.

The text between the two is exact: every depth here starts as a whole number (a trimmed graph's depths are path-step counts) and
apply_bridges only subtracts 1 (clamped at 0) or sets sequences.len(), so every depth written is a whole number below 2^53 whose "{:.2}"
text parses back to the same f64 (asserted in _gfa_text).  Links keep their order through the round trip (L lines are written per unitig in
list order and read back in file order); the re-loaded prev lists are in L-line order, and merge_linear_paths reads them only as sets.

FAST_DP (golden generation only): global_alignment_distance by rows with numpy, where the insert step is a running minimum of
X[j] - C[j] (C = prefix sums of path b's weights).  It is used only when sum(weights of a) + sum(weights of b) < 2^32: every cell is at
most the cost of the all-gaps alignment, so no u32 sum wraps and int64 arithmetic gives the same bits.  test_resolve.py checks it
against the literal DP on random cases."""
import numpy as np

import oracle_lib

U32 = 0xFFFFFFFF
FAST_DP = False
_dp_cache = {}


def reverse_path(p):   # misc.rs:443-445
    return [-u for u in reversed(p)]


def global_alignment_distance(a, b, weights):   # resolve.rs:387-418
    if FAST_DP:
        key = (tuple(a), tuple(b))
        if key not in _dp_cache:
            _dp_cache[key] = global_alignment_distance_rows(a, b, weights)
        return _dp_cache[key]
    if WRAP_DP:
        key = min((tuple(a), tuple(b)), (tuple(b), tuple(a)))      # D(a, b) == D(b, a): checked against the cell form in the tests
        if key not in _wrap_cache:
            _wrap_cache[key] = global_alignment_distance_diagonals(a, b, weights)
        return _wrap_cache[key]
    return global_alignment_distance_cells(a, b, weights)


WRAP_DP = False          # tests only: the anti-diagonal form below, exact with wraparound, for bridges of hundreds of unitigs
_wrap_cache = {}


def global_alignment_distance_diagonals(a, b, weights):
    """The cell form one anti-diagonal (i + j = d) at a time: a cell needs only the two diagonals before it, so each diagonal is a few
    uint32 vector adds and mins on the same operands as the cell form, wrapping as it does."""
    n, m = len(a), len(b)
    wa = np.array([weights[abs(u)] for u in a], dtype=np.uint32)
    wb = np.array([weights[abs(u)] for u in b], dtype=np.uint32)
    av, bv = np.array(a, dtype=np.int64), np.array(b, dtype=np.int64)
    diags = [np.zeros(n + 1, dtype=np.uint32) for _ in range(3)]       # diagonal d lives in diags[d % 3], indexed by row i
    for d in range(1, n + m + 1):
        cur, prev, prev2 = diags[d % 3], diags[(d - 1) % 3], diags[(d - 2) % 3]
        if d <= m:
            cur[0] = (int(prev[0]) + int(wb[d - 1])) & U32                # top edge: gaps in a
        if d <= n:
            cur[d] = (int(prev[d - 1]) + int(wa[d - 1])) & U32            # left edge: gaps in b
        lo, hi = max(1, d - m), min(d - 1, n)
        if lo <= hi:
            i = np.arange(lo, hi + 1)
            j = d - i
            wi, wj = wa[i - 1], wb[j - 1]
            sub = np.where(av[i - 1] == bv[j - 1], np.uint32(0), np.maximum(wi, wj))
            cur[lo:hi + 1] = np.minimum(np.minimum(prev2[i - 1] + sub, prev[i - 1] + wi), prev[i] + wj)
    return int(diags[(n + m) % 3][n])


def global_alignment_distance_cells(a, b, weights):
    n, m = len(a), len(b)
    prev = [0] * (m + 1)
    curr = [0] * (m + 1)
    for j in range(1, m + 1):
        prev[j] = (prev[j - 1] + weights[abs(b[j - 1])]) & U32
    for i in range(1, n + 1):
        wi = weights[abs(a[i - 1])]
        curr[0] = (prev[0] + wi) & U32
        for j in range(1, m + 1):
            wj = weights[abs(b[j - 1])]
            sub = 0 if a[i - 1] == b[j - 1] else max(wi, wj)
            curr[j] = min((prev[j - 1] + sub) & U32, (prev[j] + wi) & U32, (curr[j - 1] + wj) & U32)
        prev, curr = curr, prev
    return prev[m]


def global_alignment_distance_rows(a, b, weights):
    wa = np.array([weights[abs(u)] for u in a], dtype=np.int64)
    wb = np.array([weights[abs(u)] for u in b], dtype=np.int64)
    assert int(wa.sum()) + int(wb.sum()) <= U32, "the row form needs sums below 2^32"
    bv = np.array(b, dtype=np.int64)
    C = np.concatenate([[0], np.cumsum(wb)])
    prev = C.copy()
    for i in range(len(a)):
        sub = np.where(bv == a[i], 0, np.maximum(wa[i], wb))
        x = np.minimum(prev[:-1] + sub, prev[1:] + wa[i])            # match/mismatch and delete for columns 1..m
        row0 = prev[0] + wa[i]
        acc = np.minimum.accumulate(np.concatenate([[row0], x - C[1:]]))   # curr[j] - C[j] = min(x[j] - C[j], curr[j-1] - C[j-1])
        prev = acc + C
    return int(prev[-1])


def consensus_weight(header):   # sequence.rs:104-109
    key = "autocycler_consensus_weight="
    for tok in header.lower().split():
        if tok.startswith(key):
            v = tok[len(key):]
            d = v[1:] if v.startswith("+") else v
            if d and all(c in "0123456789" for c in d) and int(d) < 2 ** 64:
                return int(d)
    return 1


class Bridge:
    def __init__(self, start, end, all_paths, weights):   # resolve.rs:430-462, the ordered P^2 loop
        trimmed = [list(p[1:-1]) for p in all_paths]
        best, best_total = [], U32
        self.totals = []
        for i, pi in enumerate(trimmed):
            total = 0
            for j, pj in enumerate(trimmed):
                if i == j:
                    continue
                total = (total + global_alignment_distance(pi, pj, weights)) & U32
            self.totals.append(total)
            if total < best_total or (total == best_total and pi < best):
                best_total, best = total, list(pi)
        self.start, self.end, self.all_paths, self.best_path, self.conflicting = start, end, trimmed, best, False

    def rev_start(self):
        return -self.end

    def rev_end(self):
        return -self.start

    def depth(self):
        return len(self.all_paths)

    def key(self):   # Ord (:506-514)
        return (abs(self.start), -self.start, abs(self.end), -self.end, self.best_path)


def get_anchor_to_anchor_paths(sequence_paths, anchor_set):   # :344-365
    out = []
    for path in sequence_paths:
        last = None
        for i, value in enumerate(path):
            if abs(value) in anchor_set:
                if last is not None:
                    fwd = list(path[last:i + 1])
                    rev = reverse_path(fwd)
                    out.append(fwd if fwd > rev else rev)
                last = i
    return out


def group_paths_by_start_end(paths):   # :368-377
    groups = {}
    for p in paths:
        if p:
            groups.setdefault((p[0], p[-1]), []).append(p)
    return groups


def determine_ambiguity(bridges):   # :193-220
    sc, ec = {}, {}
    for b in bridges:
        sc[b.start] = sc.get(b.start, 0) + 1
        sc[b.rev_start()] = sc.get(b.rev_start(), 0) + 1
        ec[b.end] = ec.get(b.end, 0) + 1
        ec[b.rev_end()] = ec.get(b.rev_end(), 0) + 1
    n = 0
    for b in bridges:
        b.conflicting = sc[b.start] > 1 or sc[b.rev_start()] > 1 or ec[b.end] > 1 or ec[b.rev_end()] > 1
        n += b.conflicting
    return n


def cull_ambiguity(bridges):   # :285-313, the literal loop
    order = lambda b: (b.depth(), b.key())
    ambi = sorted([b for b in bridges if b.conflicting], key=order)
    count = 0
    while ambi:
        c = ambi[0]
        bridges.pop(next(i for i, b in enumerate(bridges) if b.start == c.start and b.end == c.end))
        count += 1
        determine_ambiguity(bridges)
        ambi = sorted([b for b in bridges if b.conflicting], key=order)
    return count


# ---- the graph ----------------------------------------------------------------------------------------------------------------------

COLOURS = {"steelblue": "Consentig", "forestgreen": "Anchor", "pink": "Bridge"}
TAG = {"Consentig": "\tCL:Z:steelblue", "Anchor": "\tCL:Z:forestgreen", "Bridge": "\tCL:Z:pink", "Other": ""}


def _lines(text):
    return [ln[:-1] if ln.endswith("\r") else ln for ln in text.split("\n") if ln]


def _parse_path(text):
    return [int(s[:-1]) * (1 if s[-1] == "+" else -1) for s in text.split(",")] if text else []


class Graph:
    """UnitigGraph::from_gfa_lines (unitig_graph.rs:55-174) minus positions: unitigs in segment order, lists of signed numbers."""

    def __init__(self, text):
        self.k = 0
        self.order, self.u = [], {}
        self.seqs = []                                      # (id, header, path)
        for ln in _lines(text):
            p = ln.split("\t")
            if p[0] == "H":
                for x in p:
                    if x.startswith("KM:i:"):
                        self.k = int(x[5:])
                        break
            elif p[0] == "S":
                num = int(p[1])
                depth = float(next(x for x in p if x.startswith("DP:f:"))[5:])
                t = "Other"
                for colour in ("steelblue", "forestgreen", "pink"):   # consentig, else anchor, else bridge
                    if f"CL:Z:{colour}" in p:
                        t = COLOURS[colour]
                        break
                self.order.append(num)
                self.u[num] = {"seq": p[2], "depth": depth, "type": t, "next": {1: [], -1: []}, "prev": {1: [], -1: []}}
            elif p[0] == "L":
                a, b = int(p[1]) * (1 if p[2] == "+" else -1), int(p[3]) * (1 if p[4] == "+" else -1)
                self._one_way(a, b)
            elif p[0] == "P":
                hd = next(x for x in p if x.startswith("HD:Z:"))[5:]
                self.seqs.append((int(p[1]), hd, _parse_path(p[2])))

    def _one_way(self, a, b):
        self.u[abs(a)]["next"][1 if a > 0 else -1].append(b)
        self.u[abs(b)]["prev"][1 if b > 0 else -1].append(a)

    def _delete_one_way(self, a, b):   # unitig_graph.rs:826-865
        nl = self.u[abs(a)]["next"][1 if a > 0 else -1]
        nl[:] = [x for x in nl if x != b]
        pl = self.u[abs(b)]["prev"][1 if b > 0 else -1]
        pl[:] = [x for x in pl if x != a]

    def delete_link(self, a, b):
        self._delete_one_way(a, b)
        self._delete_one_way(-b, -a)

    def delete_outgoing_links(self, s):
        for n in list(self.u[abs(s)]["next"][1 if s > 0 else -1]):
            self.delete_link(s, n)

    def delete_incoming_links(self, s):
        for p in list(self.u[abs(s)]["prev"][1 if s > 0 else -1]):
            self.delete_link(p, s)

    def create_link(self, a, b):   # :867-872
        self._one_way(a, b)
        if a != -b:
            self._one_way(-b, -a)

    def seq_of(self, s):
        f = self.u[abs(s)]["seq"]
        return f if s > 0 else f[::-1].translate(str.maketrans("ACGT", "TGCA"))

    def connected_components(self):   # :905-919
        seen, comps = set(), []
        for num in self.order:
            if num in seen:
                continue
            comp, stack = [], [num]
            while stack:
                c = stack.pop()
                if c in seen:
                    continue
                seen.add(c)
                comp.append(c)
                u = self.u[c]
                for lst in (u["next"][1], u["prev"][1], u["next"][-1], u["prev"][-1]):
                    for x in lst:
                        if abs(x) not in seen:
                            stack.append(abs(x))
            comps.append(sorted(comp))
        return sorted(comps)

    def remove(self, nums):   # retain + delete_dangling_links
        self.order = [n for n in self.order if n not in nums]
        for n in nums:
            del self.u[n]
        for n in self.order:
            for d in ("next", "prev"):
                for s in (1, -1):
                    self.u[n][d][s] = [x for x in self.u[n][d][s] if abs(x) in self.u]

    def gfa_text(self, other_colour=False):   # save_gfa without sequences (:317-331)
        out = [f"H\tVN:Z:1.0\tKM:i:{self.k}"]
        for n in self.order:
            d = self.u[n]["depth"]
            assert d == int(d) and abs(d) < 2 ** 53, "a depth that is not a whole number would not survive the text round trip"
            tag = TAG[self.u[n]["type"]] or ("\tCL:Z:orangered" if other_colour else "")
            out.append(f"S\t{n}\t{self.u[n]['seq']}\tDP:f:{d:.2f}{tag}")
        for n in self.order:
            for s, sign in ((1, "+"), (-1, "-")):
                for b in self.u[n]["next"][s]:
                    out.append(f"L\t{n}\t{sign}\t{abs(b)}\t{'+' if b > 0 else '-'}\t0M")
        return "\n".join(out) + "\n"


def find_anchors(g):   # :134-163
    all_ids = sorted(sid for sid, _, _ in g.seqs)
    ids = {n: [] for n in g.order}
    for sid, _, path in g.seqs:
        for s in path:
            ids[abs(s)].append(sid)
    return [n for n in g.order if sorted(ids[n]) == all_ids]


def create_bridges(g, anchors):   # :166-190
    sequence_paths = []
    for sid, hd, path in g.seqs:
        sequence_paths.extend([path] * consensus_weight(hd))
    groups = group_paths_by_start_end(get_anchor_to_anchor_paths(sequence_paths, set(anchors)))
    weights = {n: len(g.u[n]["seq"]) for n in g.order}
    bridges = [Bridge(s, e, paths, weights) for (s, e), paths in groups.items()]
    bridges.sort(key=Bridge.key)
    return bridges


def apply_bridges(g, bridges, bridge_depth):   # :223-251
    for b in bridges:
        if b.conflicting:
            continue
        g.delete_outgoing_links(b.start)
        g.delete_incoming_links(b.end)
        if not b.best_path:
            g.create_link(b.start, b.end)
            continue
        seq = "".join(g.seq_of(s) for s in b.best_path)
        num = max(g.order) + 1
        g.order.append(num)
        g.u[num] = {"seq": seq, "depth": float(bridge_depth), "type": "Bridge", "next": {1: [], -1: []}, "prev": {1: [], -1: []}}
        for p in b.all_paths:                                # reduce_depths (:261-270)
            for s in p:
                u = g.u[abs(s)]
                u["depth"] = max(0.0, u["depth"] - 1.0)
        g.create_link(b.start, num)
        g.create_link(num, b.end)
    no_anchor = set()
    for comp in g.connected_components():
        if all(g.u[n]["type"] != "Anchor" for n in comp):
            no_anchor.update(comp)
    g.remove(no_anchor)
    g.remove({n for n in g.order if not g.u[n]["depth"] > 0.0})


def _merge(text):   # merge_after_bridging (:254-258) + save_gfa
    return oracle_lib.gfa_merge_linear_paths(text, use_paths=False, renumber=True)


def _other_colour(text):   # save_gfa(.., use_other_colour = true): Other unitigs get CL:Z:orangered
    out = []
    for ln in _lines(text):
        if ln.startswith("S\t") and not any(x.startswith("CL:Z:") for x in ln.split("\t")[3:]):
            ln += "\tCL:Z:orangered"
        out.append(ln)
    return "\n".join(out) + "\n"


def resolve_gfa(trimmed_text, info=None):
    """resolve.rs:41-67 on the text of 2_trimmed.gfa -> (3_bridged.gfa, 4_merged.gfa, 5_final.gfa)."""
    g = Graph(trimmed_text)
    anchors = find_anchors(g)
    for n in anchors:
        g.u[n]["type"] = "Anchor"
    bridges = create_bridges(g, anchors)
    bridge_depth = len(g.seqs)
    conflicting = determine_ambiguity(bridges)
    apply_bridges(g, bridges, bridge_depth)
    bridged = g.gfa_text()
    merged = _merge(bridged)
    culled = cull_ambiguity(bridges)
    if culled > 0:
        g2 = Graph(trimmed_text)
        for n in anchors:
            g2.u[n]["type"] = "Anchor"
        apply_bridges(g2, bridges, bridge_depth)
        final = _other_colour(_merge(g2.gfa_text()))
    else:
        final = _other_colour(merged)
    if info is not None:
        info.update(anchors=len(anchors), conflicting=conflicting, culled=culled, bridges=len(bridges) + culled)
    return bridged, merged, final


# ---- combine ----------------------------------------------------------------------------------------------------------------------

def _topology(g):   # unitig_graph.rs:527-545
    if not g.order:
        return "empty"
    if len(g.order) > 1:
        return "fragmented"
    n = g.order[0]
    u = g.u[n]
    if not any(u["next"][1]) and not any(u["next"][-1]):
        return "linear-open-open"
    if _circular(g, n):
        return "circular"
    hs = u["next"][-1] == [n]
    he = u["next"][1] == [-n]
    os_, oe = not u["next"][-1], not u["next"][1]
    if hs and he:
        return "linear-hairpin-hairpin"
    if (hs and oe) or (os_ and he):
        return "linear-open-hairpin"
    return "other"


def _circular(g, n):   # unitig.rs:275-281
    u = g.u[n]
    return u["next"][1] == [n] and u["prev"][1] == [n]


def _linear(g, n):     # :283-292
    u = g.u[n]
    if len(u["next"][1]) > 1 or len(u["prev"][1]) > 1 or _circular(g, n):
        return False
    return all(x == -n for x in u["next"][1]) and all(x == -n for x in u["prev"][1]) and all(x == n for x in u["next"][-1]) and \
        all(x == n for x in u["prev"][-1])


def combine_gfas(texts):
    """combine.rs:90-137 -> (consensus_assembly.gfa, .fasta, .yaml)."""
    gfa, fasta, clusters = ["H\tVN:Z:1.0"], [], []
    bases = unitigs = offset = 0
    fully = True
    for text in texts:
        g = Graph(text)
        for n in g.order:
            u = g.u[n]
            tag = TAG[u["type"]] or "\tCL:Z:orangered"
            gfa.append(f"S\t{n + offset}\t{u['seq']}\tDP:f:{u['depth']:.2f}{tag}")
            topo = " circular=true topology=circular" if _circular(g, n) else " circular=false topology=linear" if _linear(g, n) else ""
            fasta.append(f">{n + offset} length={len(u['seq'])}{topo}")
            fasta.append(u["seq"])
        for n in g.order:
            for s, sign in ((1, "+"), (-1, "-")):
                for b in g.u[n]["next"][s]:
                    gfa.append(f"L\t{n + offset}\t{sign}\t{abs(b) + offset}\t{'+' if b > 0 else '-'}\t0M")
        offset += max(g.order, default=0)
        length = sum(len(g.u[n]["seq"]) for n in g.order)
        bases += length
        unitigs += len(g.order)
        clusters.append((length, len(g.order), _topology(g)))
        if len(g.order) > 1:
            fully = False
    yaml = f"consensus_assembly_bases: {bases}\nconsensus_assembly_unitigs: {unitigs}\n" \
           f"consensus_assembly_fully_resolved: {'true' if fully else 'false'}\nconsensus_assembly_clusters:"
    yaml += " []\n" if not clusters else "\n" + "".join(f"- length: {a}\n  unitigs: {b}\n  topology: {c}\n" for a, b, c in clusters)
    return "\n".join(gfa) + "\n", "".join(x + "\n" for x in fasta), yaml
