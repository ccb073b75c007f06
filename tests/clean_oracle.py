"""CPU oracle of `autocycler clean`, `autocycler gfa2fasta` and `autocycler table`: a literal Python restatement of the graph edits
(unitig_graph.rs:547-721) on per-strand lists of signed numbers, of save_graph_to_fasta (gfa2fasta.rs:55-82), and of table's file
selection, YAML values and formatting (table.rs:24-204, misc.rs:373-386).  merge_linear_paths, renumbering and the saved text go through
the C++ oracle (oracle_lib.gfa_merge_linear_paths), as resolve_oracle.py does it."""
import math
import os

import numpy as np

import oracle_lib
import resolve_oracle as R

TYPE_TAG = {"Consentig": "\tCL:Z:steelblue", "Anchor": "\tCL:Z:forestgreen", "Bridge": "\tCL:Z:pink", "Other": "\tCL:Z:orangered"}


# ---- the graph edits --------------------------------------------------------------------------------------------------------------

def remove_unitigs(g, nums):   # unitig_graph.rs:588-592
    g.remove(set(nums) & set(g.u))


def _add(g, num, seq, depth, t, positions):
    g.order.append(num)
    g.u[num] = {"seq": seq, "depth": depth, "type": t, "next": {1: [], -1: []}, "prev": {1: [], -1: []}, "positions": positions}


def _load(text):
    """The graph with each unitig's forward_positions.len(): the sequence path steps through it (unitig_graph.rs:151-174)."""
    g = R.Graph(text)
    for n in g.order:
        g.u[n]["positions"] = 0
    for _, _, path in g.seqs:
        for s in path:
            g.u[abs(s)]["positions"] += 1
    return g


def duplicate_unitig(g, num):   # :594-668
    u = g.u[num]
    links = [x for x in u["next"][1] if abs(x) != num] + [x for x in u["next"][-1] if abs(x) != num]
    if len(links) != 2:
        raise ValueError(f"unitig {num} does not contain exactly two non-self links")
    fwd, rev = list(u["next"][1]), list(u["next"][-1])
    a = max(g.order) + 1
    b = a + 1
    _add(g, a, u["seq"], u["depth"] / 2.0, u["type"], u["positions"])   # clones: the positions too
    _add(g, b, u["seq"], u["depth"] / 2.0, u["type"], u["positions"])
    remove_unitigs(g, {num})
    for x in fwd:
        if abs(x) == num:
            g.create_link(a, a if x > 0 else -a)
            g.create_link(b, b if x > 0 else -b)
    for x in rev:
        if abs(x) == num:
            g.create_link(-a, a if x > 0 else -a)
            g.create_link(-b, b if x > 0 else -b)
    non_self = [(num, x) for x in fwd if abs(x) != num] + [(-num, x) for x in rev if abs(x) != num]

    def find_replace(t, find, rep):   # misc.rs:509-515
        return tuple(rep * (1 if v > 0 else -1) if abs(v) == find else v for v in t)
    g.create_link(*find_replace(non_self[0], num, a))
    g.create_link(*find_replace(non_self[1], num, b))


def remove_low_depth_unitigs(g, min_depth):   # :670-721
    if not g.order:
        return
    for idx in reversed(range(len(g.order))):
        if idx >= len(g.order):
            continue
        num = g.order[idx]
        u = g.u[num]
        if u["depth"] > min_depth:
            continue
        ok = True
        for x in list(u["next"][1]):
            if abs(x) == num:
                continue
            if not any(abs(lk) != num for lk in g.u[abs(x)]["prev"][1 if x > 0 else -1]):
                ok = False
                break
        if ok:
            for x in list(u["prev"][1]):
                if abs(x) == num:
                    continue
                if not any(abs(lk) != num for lk in g.u[abs(x)]["next"][1 if x > 0 else -1]):
                    ok = False
                    break
        if ok:
            remove_unitigs(g, {num})


def gfa_text(g, exact=False):
    """save_gfa without P lines, use_other_colour = true.  exact: a text for the C++ oracle to load, with the depths in full precision
    and, for each position a unitig holds, a one-step P line through it."""
    out = [f"H\tVN:Z:1.0\tKM:i:{g.k}"]
    for n in g.order:
        d = g.u[n]["depth"]
        out.append(f"S\t{n}\t{g.u[n]['seq']}\tDP:f:{repr(d) if exact else format(d, '.2f')}{TYPE_TAG[g.u[n]['type']]}")
    for n in g.order:
        for s, sign in ((1, "+"), (-1, "-")):
            for b in g.u[n]["next"][s]:
                out.append(f"L\t{n}\t{sign}\t{abs(b)}\t{'+' if b > 0 else '-'}\t0M")
    if exact:
        pid = 0
        for n in g.order:
            for _ in range(g.u[n].get("positions", 0)):
                pid += 1
                out.append(f"P\t{pid}\t{n}+\tLN:i:{len(g.u[n]['seq'])}\tFN:Z:x\tHD:Z:x")
    return "\n".join(out) + "\n"


def link_count(g):   # unitig_graph.rs:478-507: (all links, links counted once)
    total = hairpins = 0
    for n in g.order:
        for s in (1, -1):
            for b in g.u[n]["next"][s]:
                total += 1
                hairpins += b == -n * s
    return total, (total - hairpins) // 2 + hairpins


def parse_tig_numbers(text):   # clean.rs:142-149
    if text is None:
        return []
    out = []
    for s in text.replace(" ", "").split(","):
        body = s[1:] if s.startswith("+") else s
        if not body or not body.isascii() or not body.isdigit() or int(body) > 0xFFFFFFFF:
            raise ValueError(f"failed to parse '{s}' as a node number")
        out.append(int(body))
    return sorted(out)


def clean(text, remove=(), duplicate=(), min_depth=None, merge=True):
    """clean.rs:26-45 on a GFA text -> the saved text."""
    g = _load(text)
    if remove:
        remove_unitigs(g, set(remove))
    for n in sorted(duplicate):
        duplicate_unitig(g, n)
    if min_depth is not None:
        remove_low_depth_unitigs(g, min_depth)
    if not merge:
        return gfa_text(g)
    return R._other_colour(oracle_lib.gfa_merge_linear_paths(gfa_text(g, exact=True), use_paths=False, renumber=True))


def qualifying_duplicates(g):
    """The unitigs duplicate_unitig accepts: exactly two non-self links over forward_next and reverse_next."""
    return [n for n in g.order if len([x for s in (1, -1) for x in g.u[n]["next"][s] if abs(x) != n]) == 2]


# ---- gfa2fasta --------------------------------------------------------------------------------------------------------------------

def gfa2fasta(text):   # gfa2fasta.rs:55-82 -> (FASTA text, (circular, linear, other))
    g = R.Graph(text)
    out, counts = [], [0, 0, 0]
    for n in g.order:
        seq = g.u[n]["seq"]
        if not seq:
            continue
        if R._circular(g, n):
            topo, counts[0] = " circular=true topology=circular", counts[0] + 1
        elif R._linear(g, n):
            topo, counts[1] = " circular=false topology=linear", counts[1] + 1
        else:
            topo, counts[2] = "", counts[2] + 1
        out.append(f">{n} length={len(seq)}{topo}\n{seq}\n")
    return "".join(out), tuple(counts)


# ---- table ------------------------------------------------------------------------------------------------------------------------

FIELD_NAMES = {  # metrics.rs:333-358
    "SubsampleMetrics": ["input_read_bases", "input_read_count", "input_read_n50", "output_reads"],
    "InputAssemblyMetrics": ["compressed_unitig_count", "compressed_unitig_total_length", "input_assemblies_count",
                             "input_assemblies_total_contigs", "input_assemblies_total_length", "input_assembly_details"],
    "ClusteringMetrics": ["cluster_balance_score", "cluster_tightness_score", "fail_cluster_count", "fail_contig_count", "fail_contig_fraction",
                          "overall_clustering_score", "pass_cluster_count", "pass_contig_count", "pass_contig_fraction"],
    "UntrimmedClusterMetrics": ["untrimmed_cluster_distance", "untrimmed_cluster_lengths", "untrimmed_cluster_mad", "untrimmed_cluster_median",
                                "untrimmed_cluster_size"],
    "TrimmedClusterMetrics": ["trimmed_cluster_lengths", "trimmed_cluster_mad", "trimmed_cluster_median", "trimmed_cluster_size"],
    "CombineMetrics": ["consensus_assembly_bases", "consensus_assembly_clusters", "consensus_assembly_fully_resolved", "consensus_assembly_unitigs"],
}
DEFAULT_FIELDS = ("input_read_count, input_read_bases, input_read_n50, pass_cluster_count, fail_cluster_count, overall_clustering_score, "
                  "untrimmed_cluster_size, untrimmed_cluster_distance, trimmed_cluster_size, trimmed_cluster_median, trimmed_cluster_mad, "
                  "consensus_assembly_bases, consensus_assembly_unitigs, consensus_assembly_fully_resolved")


class TableError(Exception):
    pass


def parse_fields(text):   # table.rs:43-60
    fields = text.replace(" ", "").split(",")
    valid = {f for names in FIELD_NAMES.values() for f in names}
    for f in fields:
        if f not in valid:
            raise TableError(f"{f} is not a valid field name")
    return fields


def powi(a, b):   # compiler-rt __powidf2
    recip, r = b < 0, 1.0
    while True:
        if b & 1:
            r *= a
        b = int(b / 2)
        if b == 0:
            break
        a *= a
    return 1 / r if recip else r


def _as_i32(x):   # `as i32`, saturating
    if math.isnan(x):
        return 0
    return int(max(-2 ** 31, min(2 ** 31 - 1, x)))


def _round(x):   # f64::round: half away from zero
    if not math.isfinite(x):
        return x
    t = float(math.trunc(x))
    return t + math.copysign(1.0, x) if abs(x - t) >= 0.5 else t


def format_float_sigfigs(value, sigfigs):   # misc.rs:373-386
    if value == 0.0:
        return f"{0.0:.{sigfigs - 1}f}"
    decimals = sigfigs - _as_i32(math.floor(math.log10(abs(value))) if math.isfinite(value) else (math.inf if math.isinf(value) else math.nan)) - 1
    factor = powi(10.0, decimals)
    with np.errstate(all="ignore"):
        rounded = float(np.float64(_round(value * factor)) / np.float64(factor)) if factor != 0 else math.nan
    if math.isnan(rounded):
        return "NaN"
    if math.isinf(rounded):
        return "inf" if rounded > 0 else "-inf"
    if decimals > 0:
        return f"{rounded:.{decimals}f}"
    return np.format_float_positional(rounded, unique=True, trim="-")


def format_value(v, sigfigs):   # table.rs:158-194
    if isinstance(v, bool):
        return "true" if v else "false"
    if isinstance(v, int):
        return str(v)
    if isinstance(v, float):
        return format_float_sigfigs(v, sigfigs)
    if isinstance(v, str):
        return v
    if isinstance(v, list):
        return "[" + ",".join(format_value(x, sigfigs) for x in v) + "]"
    if isinstance(v, tuple):   # a mapping: ((key, value), ...) in file order
        return "{" + ",".join(f"{format_value(k, sigfigs)}:{format_value(x, sigfigs)}" for k, x in v) + "}"
    return ""


def _scalar(s):   # serde_yaml's resolution of a plain scalar
    if s in ("", "~", "null", "Null", "NULL"):
        return None
    if s in ("true", "True", "TRUE"):
        return True
    if s in ("false", "False", "FALSE"):
        return False
    t = s[1:] if s[:1] in "+-" else s
    leading_zero = len(t) > 1 and t[0] == "0" and t[1:].isascii() and t[1:].isdigit()   # YAML 1.2: a string
    if not leading_zero and not (s[:1] == "+" and s[1:2] in ("+", "-")):
        t = s[1:] if s[:1] in "+-" else s
        if t.isascii() and t.isdigit():
            v = -int(t) if s[0] == "-" else int(t)
            if -2 ** 63 <= v < 2 ** 64:
                return v
        for prefix, base in (("0x", 16), ("0o", 8), ("0b", 2)):
            if t.startswith(prefix) and len(t) > 2:
                try:
                    v = int(t[2:], base)
                except ValueError:
                    break
                v = -v if s[0] == "-" else v
                if -2 ** 63 <= v < 2 ** 64:
                    return v
        u = s[1:] if s.startswith("+") else s
        if u in (".inf", ".Inf", ".INF"):
            return math.inf
        if s in ("-.inf", "-.Inf", "-.INF"):
            return -math.inf
        if s in (".nan", ".NaN", ".NAN"):
            return math.nan
        import re
        if re.fullmatch(r"-?(\d+\.?\d*|\.\d+)([eE][+-]?\d+)?", u):
            f = float(u)
            if math.isfinite(f):
                return f
    return s


def _inline(t):
    t = t.rstrip(" ")
    if t == "[]":
        return []
    if t == "{}":
        return ()
    if t[:1] == "'":
        assert t.endswith("'") and len(t) >= 2
        return t[1:-1].replace("''", "'")
    if t[:1] == '"':
        assert t.endswith('"') and len(t) >= 2
        return bytes(t[1:-1], "utf-8").decode("unicode_escape")
    assert t[:1] not in ("[", "{", "|", ">", "&", "*", "!"), t
    return _scalar(t)


def _split(t):
    if t[:1] in ("'", '"'):
        q = t[0]
        i = 1
        while True:
            if t[i] == q and q == "'" and t[i + 1:i + 2] == "'":
                i += 2
                continue
            if t[i] == q and (q == "'" or t[i - 1] != "\\"):
                break
            i += 1
        key = _inline(t[:i + 1])
        rest = t[i + 1:].lstrip(" ")
        assert rest.startswith(":")
        return key, rest[2:] if len(rest) > 1 else ""
    for i, c in enumerate(t):
        if c == ":" and (i + 1 == len(t) or t[i + 1] == " "):
            return _scalar(t[:i].rstrip(" ")), t[i + 2:]
    return None


def _is_item(t):
    return t == "-" or t.startswith("- ")


def load_yaml_map(path):
    """serde_yaml::from_str::<HashMap<String, Value>> of the block YAML the tools write -> [(key, value)] in file order; a mapping
    value is a tuple of (key, value) pairs."""
    lines = []
    for ln in open(path, encoding="utf-8").read().split("\n"):
        ln = ln[:-1] if ln.endswith("\r") else ln
        body = ln.lstrip(" ").rstrip(" \t")
        if body and not body.startswith("#") and not (body == "---" and ln[0] != " "):
            lines.append([len(ln) - len(ln.lstrip(" ")), body])
    pos = [0]

    def block(ind):
        return seq(ind) if _is_item(lines[pos[0]][1]) else mapping(ind)

    def nested(ind, same):
        if pos[0] < len(lines) and lines[pos[0]][0] > ind:
            return block(lines[pos[0]][0])
        if same and pos[0] < len(lines) and lines[pos[0]][0] == ind and _is_item(lines[pos[0]][1]):
            return seq(ind)
        return None

    def seq(ind):
        out = []
        while pos[0] < len(lines) and lines[pos[0]][0] == ind and _is_item(lines[pos[0]][1]):
            item = lines[pos[0]][1][2:]
            lead = len(item) - len(item.lstrip(" "))
            body = item[lead:]
            if not body:
                pos[0] += 1
                out.append(nested(ind, False))
            elif _is_item(body) or _split(body) is not None:
                lines[pos[0]] = [ind + 2 + lead, body]
                out.append(block(ind + 2 + lead))
            else:
                pos[0] += 1
                out.append(_inline(body))
        assert not (pos[0] < len(lines) and lines[pos[0]][0] > ind)
        return out

    def mapping(ind):
        out = []
        while pos[0] < len(lines) and lines[pos[0]][0] == ind and not _is_item(lines[pos[0]][1]):
            kv = _split(lines[pos[0]][1])
            assert kv is not None
            pos[0] += 1
            key, rest = kv
            assert all(k != key for k, _ in out)
            rest = rest.lstrip(" ")
            out.append((key, nested(ind, True) if not rest else _inline(rest)))
        assert not (pos[0] < len(lines) and lines[pos[0]][0] > ind)
        return tuple(out)

    try:
        assert lines and lines[0][0] == 0 and not _is_item(lines[0][1])
        if len(lines) == 1 and lines[0][1] == "{}":
            return []
        m = mapping(0)
        assert pos[0] == len(lines)
        assert all(isinstance(k, (str, int)) for k, _ in m)
    except (AssertionError, IndexError, UnicodeDecodeError):
        raise TableError("Failed to parse YAML file")
    return [(k if isinstance(k, str) else (("true" if k else "false") if isinstance(k, bool) else str(k)), v) for k, v in m]


def find_all_yaml_files(d):   # table.rs:118-138, sorted component by component as PathBuf sorts
    out = []

    def visit(p):
        try:
            names = os.listdir(p)
        except OSError:
            return
        for n in names:
            q = p + n if p.endswith("/") else p + "/" + n
            if os.path.isdir(q):
                visit(q)
            elif n.rfind(".") > 0 and n[n.rfind(".") + 1:] == "yaml":
                out.append(q)
    visit(d)
    return sorted(out, key=lambda p: [c for i, c in enumerate(p.split("/")) if c and not (c == "." and i > 0)])


def get_one_copy_yaml(files, name, warnings=None):   # table.rs:141-155
    found = [f for f in files if f.rsplit("/", 1)[-1] == name]
    if not found and warnings is not None:
        warnings.append(f"Warning: {name} not found")
    if len(found) > 1:
        raise TableError(f"Multiple {name} files found")
    return found[0] if found else None


def get_multi_copy_yaml(files, name, warnings=None):   # :158-168
    found = [f for f in files if f.rsplit("/", 1)[-1] == name and "/qc_fail/" not in f]
    if not found and warnings is not None:
        warnings.append(f"Warning: {name} not found")
    return found


def table(autocycler_dir=None, name="", fields=DEFAULT_FIELDS, sigfigs=3, warnings=None):
    """table.rs:24-115 -> the printed line, newline included."""
    if sigfigs == 0:
        raise TableError("--sigfigs must be 1 or greater")
    fields = parse_fields(fields)
    if autocycler_dir is None:
        return "name\t" + "\t".join(fields) + "\n"
    if "\t" in name:
        raise TableError("--name cannot contain tab characters")
    files = find_all_yaml_files(autocycler_dir)
    singles = [get_one_copy_yaml(files, f, warnings) for f in ("subsample.yaml", "input_assemblies.yaml", "clustering.yaml", "consensus_assembly.yaml")]
    multis = [get_multi_copy_yaml(files, f, warnings) for f in ("1_untrimmed.yaml", "2_trimmed.yaml")]
    values = {}
    for p in singles:
        if p:
            values.update(load_yaml_map(p))
    for group in multis:
        combined = {}
        for p in group:
            for k, v in load_yaml_map(p):
                combined.setdefault(k, []).append(v)
        values.update(combined)
    return name + "".join("\t" + (format_value(values[f], sigfigs) if f in values else "") for f in fields) + "\n"
