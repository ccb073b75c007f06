"""CPU oracle of `autocycler trim` (rrwick/Autocycler v0.6.1, trim.rs) — test infrastructure only.

A restatement of trim.rs:36-507 in Python.  overlap_alignment keeps the whole scoring matrix as the reference does (:382) and fills it
row by row: within a row, S[i][j] = max(X[j], S[i][j-1] - w_b[j]) with X[j] = max(match, delete) is a running maximum of X[j] + C[j]
minus C[j] (C = prefix sums of the column weights); every value is a multiple of 0.5 below 2^52, so those f64 sums are exact and the
matrix is the reference's bit for bit.  `overlap_alignment_cells` is the cell-by-cell form of the same loop, for cross-checking.

The graph part (load, recalculate_depths, remove_zero_depth_unitigs with delete_dangling_links, the new paths) works on GFA text and
hands merge_linear_paths + renumber_unitigs + save_gfa to the C++ oracle (oracle_lib.gfa_merge_linear_paths), which reloads the text:
links keep their order through the round trip (L lines are written per unitig in list order and read back in file order)."""
import numpy as np

import oracle_lib

GAP = 0
NONE = -1          # usize::MAX in the reference


def reverse_path(path):   # misc.rs:443-445
    return [-u for u in reversed(path)]


def _u32(x):
    return x & 0xFFFFFFFF


def _matrix_rows(path_a, path_b, weights, k, skip_diagonal):
    n = len(path_a)
    a = np.array(path_a[:k], dtype=np.int64)
    b = np.array(path_b[n - k:], dtype=np.int64)
    wa = np.array([weights[abs(u)] for u in path_a[:k]], dtype=np.float64)
    wb = np.array([weights[abs(u)] for u in path_b[n - k:]], dtype=np.float64)
    C = np.concatenate([[0.0], np.cumsum(wb)])                       # C[j] = wb[1] + ... + wb[j] (exact: integral, < 2^53)
    S = np.full((k + 1, k + 1), -np.inf)
    S[:, 0] = 0.0
    S[0, :] = 0.0
    for i in range(1, k + 1):
        prev = S[i - 1]
        match = prev[:-1] + np.where(a[i - 1] == b, wa[i - 1], -(wa[i - 1] + wb) / 2.0)
        delete = prev[1:] - wa[i - 1]
        x = np.maximum(match, delete)
        skip = (i - 1) - (n - k) + 1 if skip_diagonal else None       # the column j with global_i == global_j (:395)
        row = np.empty(k + 1)
        row[0] = 0.0
        segments = [(1, k + 1)] if skip is None or not 1 <= skip <= k else [(1, skip), (skip + 1, k + 1)]
        if skip is not None and 1 <= skip <= k:
            row[skip] = -np.inf
        for lo, hi in segments:
            if lo >= hi:
                continue
            # S[j] + C[j] = max(X[j] + C[j], S[j-1] + C[j-1]), seeded with the cell left of the segment
            seed = row[lo - 1] + C[lo - 1]
            acc = np.maximum.accumulate(np.concatenate([[seed], x[lo - 1:hi - 1] + C[lo:hi]]))[1:]
            row[lo:hi] = acc - C[lo:hi]
        S[i] = row
    return S


def _matrix_cells(path_a, path_b, weights, k, skip_diagonal):   # trim.rs:382-407 as written
    n = len(path_a)
    S = [[-float("inf")] * (k + 1) for _ in range(k + 1)]
    for i in range(k + 1):
        S[i][0] = 0.0
        S[0][i] = 0.0
    for i in range(1, k + 1):
        for j in range(1, k + 1):
            gi, gj = i - 1, n - k + j - 1
            if skip_diagonal and gi == gj:
                continue
            wi, wj = float(weights[abs(path_a[gi])]), float(weights[abs(path_b[gj])])
            m = S[i - 1][j - 1] + (wi if path_a[gi] == path_b[gj] else -(wi + wj) / 2.0)
            S[i][j] = max(m, S[i - 1][j] - wi, S[i][j - 1] - wj)
    return np.array(S)


def overlap_alignment(path_a, path_b, weights, min_identity, max_unitigs, skip_diagonal, cells=False):
    """trim.rs:366-479 -> list of (a_unitig, a_index, b_unitig, b_index), GAP = 0, NONE = -1; [] for no alignment."""
    assert len(path_a) == len(path_b)
    n = len(path_a)
    k = min(max_unitigs, n)
    S = (_matrix_cells if cells else _matrix_rows)(path_a, path_b, weights, k, skip_diagonal)
    max_score, max_i, max_j = -float("inf"), 0, 0
    for i in range(1, k + 1):                       # strict >: the smallest i wins ties (:413-419)
        if S[i][k] > max_score:
            max_score, max_i, max_j = S[i][k], i, k
    if max_score <= 0.0:
        return []
    al = []
    i, j = max_i, max_j
    while i > 0 and j > 0:
        gi, gj = i - 1, n - k + j - 1
        if path_a[gi] == path_b[gj]:
            al.append((path_a[gi], gi, path_b[gj], gj)); i -= 1; j -= 1
        elif S[i - 1][j] >= S[i][j - 1]:
            al.append((path_a[gi], gi, GAP, NONE)); i -= 1
        else:
            al.append((GAP, NONE, path_b[gj], gj)); j -= 1
    if i > 0:                                       # the traceback hit the left edge (:459)
        return []
    al.reverse()
    a_len = _u32(sum(weights[abs(p[0])] for p in al if p[0] != GAP))
    b_len = _u32(sum(weights[abs(p[2])] for p in al if p[2] != GAP))
    mean_length = (float(a_len) + float(b_len)) / 2.0
    matches = _u32(sum(weights[abs(p[0])] for p in al if p[0] == p[2]))
    if float(matches) / mean_length < min_identity:
        return []
    return al


def find_midpoint(al, weights):   # trim.rs:482-507
    total = _u32(sum((weights[abs(p[0])] if p[0] != GAP else 0) + (weights[abs(p[2])] if p[2] != GAP else 0) for p in al))
    cumulative, best_index, best_closeness = 0, 0, 1.0
    for i, p in enumerate(al):
        if p[0] != GAP:
            cumulative = _u32(cumulative + weights[abs(p[0])])
        if p[2] != GAP:
            cumulative = _u32(cumulative + weights[abs(p[2])])
        closeness = abs(0.5 - (float(cumulative) / float(total)))
        if p[0] == p[2] and closeness < best_closeness:
            best_index, best_closeness = i, closeness
    return best_index


def trim_path_start_end(path, weights, min_identity, max_unitigs):   # trim.rs:288-296
    al = overlap_alignment(path, path, weights, min_identity, max_unitigs, True)
    if not al:
        return None
    m = find_midpoint(al, weights)
    return list(path[al[m][1]:al[m][3]])


def trim_path_hairpin_end(path, weights, min_identity, max_unitigs):   # trim.rs:299-317
    al = overlap_alignment(reverse_path(path), path, weights, min_identity, max_unitigs, False)
    if not al:
        return None
    end = 0
    while al:
        while al and al[0][0] == GAP:
            al.pop(0)
        while al and al[-1][2] == GAP:
            al.pop()
        if not al:
            break
        back = al.pop()
        assert al and back[2] == -al[0][0]
        if back[0] != GAP:
            end = back[3]
        al.pop(0)
    return list(path[:end])


def trim_path_hairpin_start(path, weights, min_identity, max_unitigs):   # trim.rs:320-326
    t = trim_path_hairpin_end(reverse_path(path), weights, min_identity, max_unitigs)
    return None if t is None else reverse_path(t)


def _median(values):   # median_isize / median_usize (misc.rs:389-406)
    if not values:
        return 0
    v = sorted(values)
    n = len(v)
    return (v[n // 2 - 1] + v[n // 2]) // 2 if n % 2 == 0 else v[n // 2]


def _mad(values):      # mad_isize / mad_usize (misc.rs:409-423)
    if not values:
        return 0
    m = _median(values)
    return _median([abs(x - m) for x in values])


def _round_usize(x):   # (x).round() as usize: half away from zero, negatives saturate to 0
    import math
    r = math.floor(abs(x) + 0.5) * (1 if x >= 0 else -1)
    return max(0, int(r))


def metrics_yaml(lengths):   # TrimmedClusterMetrics (metrics.rs:209-225) in serde_yaml 0.9 form
    y = f"trimmed_cluster_size: {len(lengths)}\n"
    y += "trimmed_cluster_lengths: []\n" if not lengths else "trimmed_cluster_lengths:\n" + "".join(f"- {x}\n" for x in lengths)
    return y + f"trimmed_cluster_median: {_median(lengths) & 0xFFFFFFFF}\ntrimmed_cluster_mad: {_mad(lengths) & 0xFFFFFFFF}\n"


def _parse_path(text):
    return [int(s[:-1]) * (1 if s[-1] == "+" else -1) for s in text.split(",")] if text else []


def _path_text(path):
    return ",".join(f"{abs(u)}{'+' if u > 0 else '-'}" for u in path)


def trim_gfa(gfa_text, min_identity=0.75, max_unitigs=5000, mad=5.0, stats=None):
    """trim.rs:43-51 on the text of 1_untrimmed.gfa -> (2_trimmed.gfa text, 2_trimmed.yaml text)."""
    lines = [ln[:-1] if ln.endswith("\r") else ln for ln in gfa_text.split("\n") if ln]
    header = [ln for ln in lines if ln.startswith("H\t")]
    segs = [ln.split("\t") for ln in lines if ln.startswith("S\t")]
    links = [ln for ln in lines if ln.startswith("L\t")]
    seqs = [ln.split("\t") for ln in lines if ln.startswith("P\t")]
    weights = {int(p[1]): len(p[2]) for p in segs}          # unitig lengths before any edit (:44)
    paths = [_parse_path(p[2]) for p in seqs]
    lengths = [int(next(x for x in p if x.startswith("LN:i:"))[5:]) for p in seqs]
    S = len(seqs)
    se, hp = [None] * S, [None] * S
    if max_unitigs > 0:
        for q, path in enumerate(paths):
            se[q] = trim_path_start_end(path, weights, min_identity, max_unitigs)
            p2 = trim_path_hairpin_start(path, weights, min_identity, max_unitigs)
            p3 = trim_path_hairpin_end(p2 if p2 is not None else path, weights, min_identity, max_unitigs)
            if p2 is not None or p3 is not None:
                hp[q] = p3 if p3 is not None else p2
    se_count, hp_count = sum(x is not None for x in se), sum(x is not None for x in hp)
    if se_count or hp_count:                                # choose_trim_type (:189-226)
        results = se if se_count >= hp_count else hp
        for q in range(S):
            if results[q] is not None:
                paths[q] = results[q]
                lengths[q] = _u32(sum(weights[abs(u)] for u in paths[q]))
    keep = [True] * S
    if mad != 0.0:                                          # exclude_outliers_in_length (:229-257)
        median, dev = _median(lengths), _mad(lengths)
        lo, hi = _round_usize(float(median) - float(dev) * mad), _round_usize(float(median) + float(dev) * mad)
        keep = [lo <= x <= hi for x in lengths]
    depth = {int(p[1]): 0 for p in segs}                    # recalculate_depths (:264)
    for q in range(S):
        if keep[q]:
            for u in paths[q]:
                depth[abs(u)] += 1
    out = list(header)
    for p in segs:                                          # remove_zero_depth_unitigs (:265)
        n = int(p[1])
        if depth[n] > 0:
            out.append("\t".join([p[0], p[1], p[2]] + [f"DP:f:{float(depth[n]):.2f}" if x.startswith("DP:f:") else x for x in p[3:]]))
    for ln in links:                                        # delete_dangling_links
        parts = ln.split("\t")
        if depth[int(parts[1])] > 0 and depth[int(parts[3])] > 0:
            out.append(ln)
    for q, p in enumerate(seqs):
        if keep[q]:
            rest = [f"LN:i:{lengths[q]}" if x.startswith("LN:i:") else x for x in p[3:]]
            out.append("\t".join([p[0], p[1], _path_text(paths[q])] + rest))
    trimmed = oracle_lib.gfa_merge_linear_paths("\n".join(out) + "\n", use_paths=True, renumber=True)   # :266-268, save_gfa
    if stats is not None:
        stats.update(paths=[len(p) for p in paths])
    return trimmed, metrics_yaml([lengths[q] for q in range(S) if keep[q]])
