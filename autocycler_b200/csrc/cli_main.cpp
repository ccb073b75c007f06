// `autocycler compress`, `autocycler decompress`, `autocycler cluster`, `autocycler trim`, `autocycler resolve`, `autocycler combine`, `autocycler dotplot`,
// `autocycler clean`, `autocycler gfa2fasta`, `autocycler table` and `autocycler subsample` with the reference's flags (main.rs:126-162), messages and exit codes
// (misc.rs:130-136: "Error: <text>" on stderr, exit 1), running the H100 path through the C ABI; `autocycler helper genome_size`,
// which departs from the reference on purpose: a k-mer depth estimate on the GPU instead of the length of a Raven assembly; and
// `autocycler depth`, read-measured contig depth (not in the reference) with the reference's helper depth filter; `autocycler qv`,
// each assembly's k-mer QV and completeness against the reads (not in the reference); `autocycler unassembled`, the reads the
// assembly does not explain (not in the reference); `autocycler polish`, the consensus corrected from the reads' k-mers (not in the
// reference); and `autocycler variants`, the alleles the reads carry beside the consensus (not in the reference).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/autocycler_gpu.h"

static const char* compress_usage =
    "Usage: autocycler compress --assemblies_dir <ASSEMBLIES_DIR> --autocycler_dir <AUTOCYCLER_DIR> [OPTIONS]\n\n"
    "Options:\n"
    "  -i, --assemblies_dir <DIR>   Directory containing input assemblies (required)\n"
    "  -a, --autocycler_dir <DIR>   Autocycler directory to be created (required)\n"
    "      --kmer <KMER>            K-mer size for De Bruijn graph [default: 51]\n"
    "      --max_contigs <N>        refuse to run if mean contigs per assembly exceeds this value [default: 25]\n"
    "  -t, --threads <THREADS>      Number of CPU threads (end repair) [default: 8]\n"
    "      --device <ORDINAL>       CUDA device [default: 0]\n"
    "      --devices <A,B,...>      several CUDA devices of this box: the assemblies are sharded by file over them\n";

// A subcommand's arguments, read one flag at a time (argv[1] is the subcommand).  Errors in them exit with 2.
struct Args {
    int argc; char** argv; const char* usage;
    int i = 1; std::string flag;
    bool next() { if (++i >= argc) return false; flag = argv[i]; return true; }
    bool is(const char* a, const char* b = nullptr) const { return flag == a || (b && flag == b); }
    const char* value() {
        if (i + 1 >= argc) { fprintf(stderr, "error: a value is required for '%s'\n", flag.c_str()); exit(2); }
        return argv[++i];
    }
    // The value as a number: all of it must parse, and an integer takes no sign.  u32: dotplot's options, which accept a '+' and
    // check the range instead, and print no usage after "invalid value".
    double number(bool integral, bool u32 = false) {
        const char* v = value();
        char* end = nullptr;
        const double x = integral ? (double)strtoul(v, &end, 10) : strtod(v, &end);
        const bool bad = u32 ? (*v == '-' || x > 0xFFFFFFFFul) : (integral && (*v == '-' || *v == '+'));
        if (!*v || *end || bad) { fprintf(stderr, "error: invalid value '%s' for '%s'\n%s", v, flag.c_str(), u32 ? "" : usage); exit(2); }
        return x;
    }
    // The value as an exact u64 (digits only, at most 2^64 - 1): a seed must not go through a double, which rounds above 2^53.
    uint64_t u64() {
        const char* v = value();
        uint64_t x = 0; bool bad = !*v;
        for (const char* q = v; *q && !bad; ++q) {
            if (*q < '0' || *q > '9' || x > (UINT64_MAX - (uint64_t)(*q - '0')) / 10) bad = true;
            else x = x * 10 + (uint64_t)(*q - '0');
        }
        if (bad) { fprintf(stderr, "error: invalid value '%s' for '%s'\n%s", v, flag.c_str(), usage); exit(2); }
        return x;
    }
    // One or more values: the flag's value and every argument after it up to the next flag
    std::vector<std::string> values() {
        std::vector<std::string> v{value()};
        while (i + 1 < argc && argv[i + 1][0] != '-') v.push_back(argv[++i]);
        return v;
    }
    int help() const { fprintf(stderr, "%s", usage); return 0; }
    int missing() const { fprintf(stderr, "%s", usage); return 2; }
    int unexpected() const { fprintf(stderr, "error: unexpected argument '%s'\n%s", flag.c_str(), usage); return 2; }
};

static std::vector<const char*> c_strings(const std::vector<std::string>& v) {
    std::vector<const char*> p;
    for (const std::string& s : v) p.push_back(s.c_str());
    return p;
}

static int finish(int rc) {
    if (rc == AC_OK) return 0;
    fprintf(stderr, "\nError: %s\n", ac_last_error(nullptr));
    return 1;
}

// `autocycler compress` (main.rs:126-148, compress.rs:32-62)
static int compress_main(int argc, char** argv) {
    Args a{argc, argv, compress_usage};
    std::string in, out; unsigned k = 51, max_contigs = 25, threads = 8; int device = 0;
    std::vector<int32_t> devices;
    while (a.next()) {
        if (a.is("-i", "--assemblies_dir")) in = a.value();
        else if (a.is("-a", "--autocycler_dir")) out = a.value();
        else if (a.is("--kmer")) k = (unsigned)strtoul(a.value(), nullptr, 10);
        else if (a.is("--max_contigs")) max_contigs = (unsigned)strtoul(a.value(), nullptr, 10);
        else if (a.is("-t", "--threads")) threads = (unsigned)strtoul(a.value(), nullptr, 10);
        else if (a.is("--device")) device = atoi(a.value());
        else if (a.is("--devices")) { devices.clear(); for (const char* q = a.value(); *q;) { devices.push_back((int32_t)strtol(q, (char**)&q, 10)); if (*q == ',') ++q; else if (*q) { fprintf(stderr, "error: --devices wants a comma-separated list of ordinals\n"); return 2; } } }
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (in.empty() || out.empty()) return a.missing();
    fprintf(stderr, "\nStarting autocycler compress (%s)\n\nSettings:\n  --assemblies_dir %s\n  --autocycler_dir %s\n  --kmer %u\n  --threads %u\n\n",
            ac_version(), in.c_str(), out.c_str(), k, threads);
    if (devices.empty()) devices.push_back(device);
    const int node = ac_bind_host_to_device(devices[0]);   // stay on the socket of the GPU that finishes the graph; harmless when the topology cannot be read
    if (node >= 0) fprintf(stderr, "host threads bound to NUMA node %d (device %d)\n\n", node, devices[0]);
    return finish(ac_compress_dir_devices(in.c_str(), out.c_str(), k, max_contigs, threads, devices.data(), (int32_t)devices.size(), 1));
}

// `autocycler decompress` (main.rs:150-162, decompress.rs:27-57); it has no -h
static int decompress_main(int argc, char** argv) {
    Args a{argc, argv, "Usage: autocycler decompress --in_gfa <IN_GFA> [--out_dir <DIR>] [--out_file <FASTA>]\n"};
    std::string in, out_dir, out_file; int device = 0;
    while (a.next()) {
        if (a.is("-i", "--in_gfa")) in = a.value();
        else if (a.is("-o", "--out_dir")) out_dir = a.value();
        else if (a.is("-f", "--out_file")) out_file = a.value();
        else if (a.is("--device")) device = atoi(a.value());
        else return a.unexpected();
    }
    if (in.empty()) return a.missing();
    fprintf(stderr, "\nStarting autocycler decompress (%s)\n\nSettings:\n  --in_gfa %s\n", ac_version(), in.c_str());
    if (!out_dir.empty()) fprintf(stderr, "  --out_dir %s\n", out_dir.c_str());
    if (!out_file.empty()) fprintf(stderr, "  --out_file %s\n", out_file.c_str());
    fprintf(stderr, "\n");
    return finish(ac_decompress_gfa(in.c_str(), out_dir.empty() ? nullptr : out_dir.c_str(), out_file.empty() ? nullptr : out_file.c_str(), device, 1));
}

// `autocycler trim` (main.rs:301-322, trim.rs:36-101): -c takes one or more cluster directories, up to the next flag, trimmed together
// (ac_trim_dirs); the library prints each directory's Starting block and report, in argument order
static int trim_main(int argc, char** argv) {
    Args a{argc, argv, "Usage: autocycler trim --cluster_dir <CLUSTER_DIR>... [--min_identity 0.75] [--max_unitigs 5000] [--mad 5.0] [--threads 8] [--device N]\n"};
    std::vector<std::string> dirs; double min_identity = 0.75, mad = 5.0; unsigned long max_unitigs = 5000, threads = 8; int device = 0;
    while (a.next()) {
        if (a.is("-c", "--cluster_dir")) dirs = a.values();
        else if (a.is("--min_identity")) min_identity = a.number(false);
        else if (a.is("--max_unitigs")) max_unitigs = (unsigned long)a.number(true);
        else if (a.is("--mad")) mad = a.number(false);
        else if (a.is("-t", "--threads")) threads = (unsigned long)a.number(true);
        else if (a.is("--device")) device = atoi(a.value());
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (dirs.empty() || dirs[0].empty()) return a.missing();
    if (max_unitigs > 0xFFFFFFFFul) max_unitigs = 0xFFFFFFFFul;
    if (threads > 0xFFFFFFFFul) threads = 0xFFFFFFFFul;
    const std::vector<const char*> ptrs = c_strings(dirs);
    return finish(ac_trim_dirs(ptrs.data(), (uint32_t)ptrs.size(), min_identity, (uint32_t)max_unitigs, mad, (uint32_t)threads, device,
                               AC_VERBOSE_REPORT | AC_VERBOSE_BANNER, nullptr));
}

// `autocycler cluster` (main.rs:92-113, cluster.rs:30-114)
static int cluster_main(int argc, char** argv) {
    Args a{argc, argv, "Usage: autocycler cluster --autocycler_dir <AUTOCYCLER_DIR> [--cutoff 0.2] [--min_assemblies N] [--max_contigs 25] [--manual 1,2,3] [--device N]\n"};
    std::string dir, manual; bool has_manual = false; double cutoff = 0.2; long long min_assemblies = -1; unsigned long max_contigs = 25; int device = 0;
    while (a.next()) {
        if (a.is("-a", "--autocycler_dir")) dir = a.value();
        else if (a.is("--cutoff")) cutoff = a.number(false);
        else if (a.is("--min_assemblies")) min_assemblies = (long long)a.number(true);
        else if (a.is("--max_contigs")) max_contigs = (unsigned long)a.number(true);
        else if (a.is("--manual")) { manual = a.value(); has_manual = true; }
        else if (a.is("--device")) device = atoi(a.value());
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (dir.empty()) return a.missing();
    if (max_contigs > 0xFFFFFFFFul) max_contigs = 0xFFFFFFFFul;
    fprintf(stderr, "\nStarting autocycler cluster (%s)\n\n", ac_version());
    return finish(ac_cluster_dir(dir.c_str(), cutoff, min_assemblies, (uint32_t)max_contigs, has_manual ? manual.c_str() : nullptr, device, 1));
}

// `autocycler resolve` (main.rs:238-247, resolve.rs:31-111): -c takes one or more cluster directories, as for trim (ac_resolve_dirs)
static int resolve_main(int argc, char** argv) {
    Args a{argc, argv, "Usage: autocycler resolve --cluster_dir <CLUSTER_DIR>... [--verbose] [--device N]\n"};
    std::vector<std::string> dirs; bool verbose = false; int device = 0;
    while (a.next()) {
        if (a.is("-c", "--cluster_dir")) dirs = a.values();
        else if (a.is("--verbose")) verbose = true;
        else if (a.is("--device")) device = atoi(a.value());
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (dirs.empty() || dirs[0].empty()) return a.missing();
    const std::vector<const char*> ptrs = c_strings(dirs);
    return finish(ac_resolve_dirs(ptrs.data(), (uint32_t)ptrs.size(), (verbose ? AC_VERBOSE_REPORT : 0) | AC_VERBOSE_BANNER, device, nullptr));
}

// `autocycler combine` (main.rs:115-124, combine.rs:25-87): -i takes one or more GFAs, up to the next flag
static int combine_main(int argc, char** argv) {
    Args a{argc, argv, "Usage: autocycler combine --autocycler_dir <AUTOCYCLER_DIR> --in_gfas <IN_GFAS>...\n"};
    std::string dir; std::vector<std::string> gfas;
    while (a.next()) {
        if (a.is("-a", "--autocycler_dir")) dir = a.value();
        else if (a.is("-i", "--in_gfas")) { const std::vector<std::string> v = a.values(); gfas.insert(gfas.end(), v.begin(), v.end()); }
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (dir.empty() || gfas.empty()) return a.missing();
    const std::vector<const char*> ptrs = c_strings(gfas);
    fprintf(stderr, "\nStarting autocycler combine (%s)\n\n", ac_version());
    return finish(ac_combine_dir(dir.c_str(), ptrs.data(), (uint32_t)ptrs.size(), 1));
}

// `autocycler dotplot` (main.rs:164-181, dotplot.rs:44-52)
static int dotplot_main(int argc, char** argv) {
    Args a{argc, argv, "Usage: autocycler dotplot --input <INPUT> --out_png <OUT_PNG> [--res <RES>] [--kmer <KMER>] [--font <TTF>] [--device N]\n"};
    std::string in, out, font; bool have_font = false; unsigned long res = 2000, kmer = 32; int device = 0;
    while (a.next()) {
        if (a.is("-i", "--input")) in = a.value();
        else if (a.is("-o", "--out_png")) out = a.value();
        else if (a.is("--res")) res = (unsigned long)a.number(true, true);
        else if (a.is("--kmer")) kmer = (unsigned long)a.number(true, true);
        else if (a.is("--font")) { font = a.value(); have_font = true; }
        else if (a.is("--device")) device = atoi(a.value());
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (in.empty() || out.empty()) return a.missing();
    fprintf(stderr, "\nStarting autocycler dotplot (%s)\n    This command will take a unitig graph (either before or after trimming) and generate a dotplot image "
                    "containing all pairwise comparisons of the sequences.\n\nSettings:\n  --input %s\n  --res %lu\n  --kmer %lu\n\n",
            ac_version(), in.c_str(), res, kmer);
    return finish(ac_dotplot_dir(in.c_str(), out.c_str(), (uint32_t)res, (uint32_t)kmer, have_font ? font.c_str() : nullptr, device, 1, nullptr));
}

// `autocycler clean` (main.rs:69-90, clean.rs:23-45); no device
static int clean_main(int argc, char** argv) {
    Args a{argc, argv, "Usage: autocycler clean --in_gfa <IN_GFA> --out_gfa <OUT_GFA> [--remove 1,2,3] [--duplicate 4,5] [--min_depth D]\n"};
    std::string in, out, remove, duplicate; bool has_remove = false, has_duplicate = false, has_min_depth = false; double min_depth = 0;
    while (a.next()) {
        if (a.is("-i", "--in_gfa")) in = a.value();
        else if (a.is("-o", "--out_gfa")) out = a.value();
        else if (a.is("-r", "--remove")) { remove = a.value(); has_remove = true; }
        else if (a.is("-d", "--duplicate")) { duplicate = a.value(); has_duplicate = true; }
        else if (a.is("-m", "--min_depth")) { min_depth = a.number(false); has_min_depth = true; }
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (in.empty() || out.empty()) return a.missing();
    return finish(ac_clean_gfa(in.c_str(), out.c_str(), has_remove ? remove.c_str() : nullptr, has_duplicate ? duplicate.c_str() : nullptr,
                               has_min_depth ? &min_depth : nullptr, 1));
}

// `autocycler gfa2fasta` (main.rs:183-192, gfa2fasta.rs:23-29); no device
static int gfa2fasta_main(int argc, char** argv) {
    Args a{argc, argv, "Usage: autocycler gfa2fasta --in_gfa <IN_GFA> --out_fasta <OUT_FASTA>\n"};
    std::string in, out;
    while (a.next()) {
        if (a.is("-i", "--in_gfa")) in = a.value();
        else if (a.is("-o", "--out_fasta")) out = a.value();
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (in.empty() || out.empty()) return a.missing();
    return finish(ac_gfa_to_fasta(in.c_str(), out.c_str(), 1));
}

// `autocycler table` (main.rs:276-299, table.rs:24-32): the line goes to stdout; no device
static int table_main(int argc, char** argv) {
    Args a{argc, argv, "Usage: autocycler table [--autocycler_dir <AUTOCYCLER_DIR>] [--name <NAME>] [--fields <FIELDS>] [--sigfigs 3]\n"};
    std::string dir, name, fields; bool has_dir = false, has_fields = false; unsigned long long sigfigs = 3;
    while (a.next()) {
        if (a.is("-a", "--autocycler_dir")) { dir = a.value(); has_dir = true; }
        else if (a.is("-n", "--name")) name = a.value();
        else if (a.is("-f", "--fields")) { fields = a.value(); has_fields = true; }
        else if (a.is("-s", "--sigfigs")) sigfigs = (unsigned long long)a.number(true);
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    uint64_t n = 0;
    const char* d = has_dir ? dir.c_str() : nullptr, *f = has_fields ? fields.c_str() : nullptr;
    int rc = ac_table_text(d, name.c_str(), f, sigfigs, 1, nullptr, 0, &n);
    std::string line(n, '\0');
    if (rc == AC_OK) rc = ac_table_text(d, name.c_str(), f, sigfigs, 0, &line[0], n, &n);
    if (rc == AC_OK) fwrite(line.data(), 1, line.size(), stdout);
    return finish(rc);
}

// `autocycler subsample` (main.rs:249-274, subsample.rs:29-43)
static int subsample_main(int argc, char** argv) {
    Args a{argc, argv, "Usage: autocycler subsample --reads <READS> --out_dir <OUT_DIR> --genome_size <GENOME_SIZE> [--count 4] [--min_read_depth 25.0] [--seed 0] [--device N]\n"};
    std::string reads, out, gsize; bool has_gsize = false; uint64_t count = 4, seed = 0; double depth = 25.0; int device = 0;
    while (a.next()) {
        if (a.is("-r", "--reads")) reads = a.value();
        else if (a.is("-o", "--out_dir")) out = a.value();
        else if (a.is("-g", "--genome_size")) { gsize = a.value(); has_gsize = true; }
        else if (a.is("-c", "--count")) count = a.u64();
        else if (a.is("-d", "--min_read_depth")) depth = a.number(false);
        else if (a.is("-s", "--seed")) seed = a.u64();
        else if (a.is("--device")) device = atoi(a.value());
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (reads.empty() || out.empty() || !has_gsize) return a.missing();
    return finish(ac_subsample_dir(reads.c_str(), out.c_str(), gsize.c_str(), count, depth, seed, device, 1, nullptr));
}

// `autocycler helper genome_size` (main.rs:194-236, helper.rs:388-403), the one helper task this build runs, and not as the reference
// does: the estimate comes from the reads' k-mer depth spectrum, counted on the GPU, instead of the total length of a Raven assembly.
// The number alone goes to stdout.  -t is accepted because the pipelines pass it; the assembler tasks' flags and --args are refused.
static const char* helper_usage =
    "Usage: autocycler helper genome_size --reads <READS> [--threads 8] [--dir <DIR>] [--kmer 21] [--device N]\n\n"
    "Estimates the genome size from the reads' canonical k-mer depth spectrum, counted on the GPU, and prints it (bases) on stdout.\n"
    "This departs from the reference, which assembles the reads with Raven and prints the assembly's total length: the numbers differ.\n"
    "A replicon present in c copies per genome counts c times, and so does each copy of a repeat.\n\n"
    "Options:\n"
    "  -r, --reads <READS>      Input long reads in FASTQ format, gzipped or not (required)\n"
    "  -t, --threads <THREADS>  Accepted for the pipelines' command lines; the counting runs on the GPU [default: 8]\n"
    "  -d, --dir <DIR>          Directory to create and write kmer_histogram.tsv into (count<TAB>k-mers)\n"
    "      --kmer <KMER>        K-mer size, odd, 11 to 31 [default: 21]\n"
    "      --device <ORDINAL>   CUDA device [default: 0]\n"
    "The other helper tasks (canu, flye, metamdbg, miniasm, myloasm, necat, nextdenovo, plassembler, raven, redbean) run external\n"
    "assemblers, which this build does not include.\n";
static int helper_main(int argc, char** argv) {
    Args a{argc, argv, helper_usage};
    if (argc < 3 || argv[2][0] == '-') {
        if (argc >= 3 && (strcmp(argv[2], "-h") == 0 || strcmp(argv[2], "--help") == 0)) return a.help();
        return a.missing();
    }
    const std::string task = argv[2];
    if (task != "genome_size") {
        fprintf(stderr, "\nError: helper task '%s' runs an external assembler, which this build does not include; only genome_size runs here\n",
                task.c_str());
        return 1;
    }
    a.i = 2;
    std::string reads, dir; bool has_dir = false; unsigned long k = 21; int device = 0;
    while (a.next()) {
        if (a.is("-r", "--reads")) reads = a.value();
        else if (a.is("-t", "--threads")) a.number(true);
        else if (a.is("-d", "--dir")) { dir = a.value(); has_dir = true; }
        else if (a.is("--kmer")) k = (unsigned long)a.number(true);
        else if (a.is("--device")) device = atoi(a.value());
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (reads.empty()) return a.missing();
    ac_genome_size_info info;
    const int rc = ac_genome_size_estimate(reads.c_str(), k > 0xFFFFFFFFul ? 0 : (uint32_t)k, device, has_dir ? dir.c_str() : nullptr, 1, nullptr, &info);
    if (rc == AC_OK) printf("%llu\n", (unsigned long long)info.estimate);
    return finish(rc);
}

// `autocycler depth`: each contig's read depth from the reads' k-mers, counted on the GPU (an addition that is not in the reference), and
// helper.rs:889-931's depth filter; with --source header, the reference's filter alone on the depths the headers carry.  Nothing goes
// to stdout.
static const char* depth_usage =
    "Usage: autocycler depth --assembly <ASSEMBLY> --out_fasta <OUT_FASTA> [--reads <READS>] [--source reads|header] [--kmer 21]\n"
    "                        [--min_depth_abs X] [--min_depth_rel Y] [--tsv <FILE>] [--device N]\n\n"
    "Measures each contig's read depth from the reads' k-mers on the GPU and appends depth=<median> to its header, then applies the\n"
    "reference's helper depth filter. Read-measured depth is not in the reference; --source header is the reference's filter alone.\n\n"
    "Options:\n"
    "  -i, --assembly <ASSEMBLY>   Input assembly in FASTA format, gzipped or not (required)\n"
    "  -o, --out_fasta <FASTA>     Output FASTA, one line per sequence (required)\n"
    "  -r, --reads <READS>         Long reads in FASTQ format, gzipped or not (required with --source reads)\n"
    "      --source <SOURCE>       reads: measure the depth from the reads; header: the depth in each header [default: reads]\n"
    "      --kmer <KMER>           K-mer size, odd, 11 to 31 [default: 21]\n"
    "      --min_depth_abs <X>     Exclude contigs with a depth less than this absolute value\n"
    "      --min_depth_rel <Y>     Exclude contigs with a depth less than this fraction of the longest contig's depth\n"
    "      --tsv <FILE>            Write name, length, unique k-mers and depth per contig\n"
    "      --device <ORDINAL>      CUDA device [default: 0]\n";
static int depth_main(int argc, char** argv) {
    Args a{argc, argv, depth_usage};
    std::string in, out, reads, tsv, source = "reads"; bool has_tsv = false, has_abs = false, has_rel = false;
    double min_abs = 0, min_rel = 0; unsigned long k = 21; int device = 0;
    while (a.next()) {
        if (a.is("-i", "--assembly")) in = a.value();
        else if (a.is("-o", "--out_fasta")) out = a.value();
        else if (a.is("-r", "--reads")) reads = a.value();
        else if (a.is("--source")) {
            source = a.value();
            if (source != "reads" && source != "header") { fprintf(stderr, "error: invalid value '%s' for '--source'\n%s", source.c_str(), depth_usage); return 2; }
        }
        else if (a.is("--kmer")) k = (unsigned long)a.number(true);
        else if (a.is("--min_depth_abs")) { min_abs = a.number(false); has_abs = true; }
        else if (a.is("--min_depth_rel")) { min_rel = a.number(false); has_rel = true; }
        else if (a.is("--tsv")) { tsv = a.value(); has_tsv = true; }
        else if (a.is("--device")) device = atoi(a.value());
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (in.empty() || out.empty() || (source == "reads" && reads.empty())) return a.missing();
    return finish(ac_depth_fasta(in.c_str(), reads.empty() ? nullptr : reads.c_str(), out.c_str(), has_tsv ? tsv.c_str() : nullptr, source == "header",
                                 k > 0xFFFFFFFFul ? 0 : (uint32_t)k, has_abs ? &min_abs : nullptr, has_rel ? &min_rel : nullptr, device, 1,
                                 nullptr, nullptr, 0, nullptr));
}

// `autocycler qv`: each assembly's k-mer QV and completeness against the reads, counted on the GPU (not in the reference).  qv.tsv also
// goes to stdout, byte for byte.
static const char* qv_usage =
    "Usage: autocycler qv --reads <READS> --assemblies <FASTA|DIR>... --out_dir <DIR> [--kmer 21] [--min_count N] [--device N]\n\n"
    "Measures each assembly's k-mer accuracy (QV) and completeness against the reads, counted on the GPU, as Merqury defines them: QV\n"
    "from the assembly k-mers the reads do not support, completeness from the reads' solid k-mers the assembly holds. This command is\n"
    "not in the reference. Writes qv.tsv (also to stdout), contig_qv.tsv, kmer_histogram.tsv, unsupported/<n>.bed and spectra_cn/<n>.tsv.\n\n"
    "Options:\n"
    "  -r, --reads <READS>            Long reads in FASTQ format, gzipped or not (required)\n"
    "  -i, --assemblies <FASTA|DIR>...  Assemblies in FASTA format, gzipped or not, or directories of them (required)\n"
    "  -o, --out_dir <DIR>            Directory to create and write the tables into (required)\n"
    "      --kmer <KMER>              K-mer size, odd, 11 to 31 [default: 21]\n"
    "      --min_count <N>            Read count from which a k-mer supports the assembly, 1 to 16383 (1: Merqury's QV)\n"
    "                                 [default: the valley of the reads' k-mer spectrum]\n"
    "      --device <ORDINAL>         CUDA device [default: 0]\n";
static int qv_main(int argc, char** argv) {
    Args a{argc, argv, qv_usage};
    std::string reads, out; std::vector<std::string> inputs; bool has_min = false; unsigned long k = 21, min_count = 0; int device = 0;
    while (a.next()) {
        if (a.is("-r", "--reads")) reads = a.value();
        else if (a.is("-i", "--assemblies")) { const std::vector<std::string> v = a.values(); inputs.insert(inputs.end(), v.begin(), v.end()); }
        else if (a.is("-o", "--out_dir")) out = a.value();
        else if (a.is("--kmer")) k = (unsigned long)a.number(true);
        else if (a.is("--min_count")) { min_count = (unsigned long)a.number(true); has_min = true; }
        else if (a.is("--device")) device = atoi(a.value());
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (reads.empty() || out.empty() || inputs.empty()) return a.missing();
    const std::vector<const char*> ptrs = c_strings(inputs);
    const uint32_t t = min_count > 0xFFFFFFFFul ? 0 : (uint32_t)min_count;
    const int rc = ac_qv_dir(reads.c_str(), ptrs.data(), (uint32_t)ptrs.size(), out.c_str(), k > 0xFFFFFFFFul ? 0 : (uint32_t)k, has_min ? &t : nullptr,
                             device, 1, nullptr, nullptr, nullptr, 0, nullptr);
    if (rc == AC_OK) {
        FILE* f = fopen((out + "/qv.tsv").c_str(), "rb");
        if (f) {
            char buf[1 << 16]; size_t n;
            while ((n = fread(buf, 1, sizeof buf, f)) > 0) fwrite(buf, 1, n, stdout);
            fclose(f);
        }
    }
    return finish(rc);
}

// `autocycler unassembled`: the reads the assembly does not explain, and the depth of the sequence it misses, counted on the GPU (not in
// the reference).  summary.tsv also goes to stdout, byte for byte.
static const char* unassembled_usage =
    "Usage: autocycler unassembled --reads <READS> --assemblies <FASTA|DIR>... --out_dir <DIR> [--kmer 21] [--min_count N] [--min_solid 100]\n"
    "                              [--min_fraction 0.5] [--device N]\n\n"
    "Finds the reads the assembly does not explain, counted on the GPU: the reads where a large share of the solid k-mers is absent from\n"
    "every input assembly, and the read depth of those absent k-mers against the genome's k-mer peak (a missing plasmid shows up as its\n"
    "copy number). This command is not in the reference. Writes unassembled.fastq, unassembled.tsv, fraction_histogram.tsv,\n"
    "absent_histogram.tsv, kmer_histogram.tsv and summary.tsv (also to stdout).\n\n"
    "Options:\n"
    "  -r, --reads <READS>            Long reads in FASTQ format, gzipped or not (required)\n"
    "  -i, --assemblies <FASTA|DIR>...  Assemblies in FASTA format, gzipped or not, or directories of them; together they are the\n"
    "                                 assembly (required)\n"
    "  -o, --out_dir <DIR>            Directory to create and write the reads and tables into (required)\n"
    "      --kmer <KMER>              K-mer size, odd, 11 to 31 [default: 21]\n"
    "      --min_count <N>            Read count from which a k-mer is solid, 1 to 16383 [default: the valley of the reads' k-mer spectrum]\n"
    "      --min_solid <N>            Solid k-mers a read needs to be scored, at least 1 [default: 100]\n"
    "      --min_fraction <F>         Share of a scored read's solid k-mers that must be absent from the assembly to select it,\n"
    "                                 above 0 and at most 1 [default: 0.5]\n"
    "      --device <ORDINAL>         CUDA device [default: 0]\n";
static int unassembled_main(int argc, char** argv) {
    Args a{argc, argv, unassembled_usage};
    std::string reads, out; std::vector<std::string> inputs; bool has_min = false;
    unsigned long k = 21, min_count = 0; double min_solid = 100, min_fraction = 0.5; int device = 0;
    auto refuse = [&]() { fprintf(stderr, "error: invalid value '%s' for '%s'\n%s", argv[a.i], a.flag.c_str(), unassembled_usage); return 2; };
    while (a.next()) {
        if (a.is("-r", "--reads")) reads = a.value();
        else if (a.is("-i", "--assemblies")) { const std::vector<std::string> v = a.values(); inputs.insert(inputs.end(), v.begin(), v.end()); }
        else if (a.is("-o", "--out_dir")) out = a.value();
        else if (a.is("--kmer")) { k = (unsigned long)a.number(true); if (k < 11 || k > 31 || k % 2 == 0) return refuse(); }
        else if (a.is("--min_count")) { min_count = (unsigned long)a.number(true); has_min = true; }
        else if (a.is("--min_solid")) { min_solid = a.number(true); if (min_solid < 1) return refuse(); }
        else if (a.is("--min_fraction")) { min_fraction = a.number(false); if (!(min_fraction > 0.0 && min_fraction <= 1.0)) return refuse(); }
        else if (a.is("--device")) device = atoi(a.value());
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (reads.empty() || out.empty() || inputs.empty()) return a.missing();
    const std::vector<const char*> ptrs = c_strings(inputs);
    const uint32_t t = min_count > 0xFFFFFFFFul ? 0 : (uint32_t)min_count;
    const uint64_t solid = min_solid >= 18446744073709551615.0 ? UINT64_MAX : (uint64_t)min_solid;
    const int rc = ac_unassembled_dir(reads.c_str(), ptrs.data(), (uint32_t)ptrs.size(), out.c_str(), (uint32_t)k, has_min ? &t : nullptr, solid,
                                      min_fraction, device, 1, nullptr);
    if (rc == AC_OK) {
        FILE* f = fopen((out + "/summary.tsv").c_str(), "rb");
        if (f) {
            char buf[1 << 16]; size_t n;
            while ((n = fread(buf, 1, sizeof buf, f)) > 0) fwrite(buf, 1, n, stdout);
            fclose(f);
        }
    }
    return finish(rc);
}

// `autocycler polish`: the consensus corrected where the reads' k-mers do not support it, with candidate edits scored on the GPU (not in
// the reference).  summary.tsv also goes to stdout, byte for byte.
static const char* polish_usage =
    "Usage: autocycler polish --reads <READS> --input <FASTA> --out_dir <DIR> [--kmer 21] [--min_count N] [--max_indel 3] [--rounds 3]\n"
    "                         [--device N]\n\n"
    "Corrects the consensus where the reads' k-mers do not support it, with candidate edits scored on the GPU: at each run of\n"
    "unsupported k-mers it tries every substitution and every insertion or deletion of up to --max_indel bases, and keeps the one that\n"
    "makes every k-mer it touches solid. This command is not in the reference. Writes polished.fasta, edits.tsv, rounds.tsv,\n"
    "remaining.bed and summary.tsv (also to stdout). Paired short reads go in as one file: cat R1.fq.gz R2.fq.gz > reads.fq.gz.\n\n"
    "Options:\n"
    "  -r, --reads <READS>            Reads in FASTQ format, gzipped or not (required)\n"
    "  -i, --input <FASTA>            Assembly in FASTA format, gzipped or not (required)\n"
    "  -o, --out_dir <DIR>            Directory to create and write the polished assembly and tables into (required)\n"
    "      --kmer <KMER>              K-mer size, odd, 11 to 31 [default: 21]\n"
    "      --min_count <N>            Read count from which a k-mer is solid, 1 to 16383 [default: the valley of the reads' k-mer spectrum]\n"
    "      --max_indel <L>            Longest insertion or deletion tried, 1 to 4 [default: 3]\n"
    "      --rounds <N>               Most rounds of edits, 1 to 10 [default: 3]\n"
    "      --device <ORDINAL>         CUDA device [default: 0]\n";
static int polish_main(int argc, char** argv) {
    Args a{argc, argv, polish_usage};
    std::string reads, in, out; bool has_min = false;
    unsigned long k = 21, min_count = 0, max_indel = 3, rounds = 3; int device = 0;
    auto refuse = [&]() { fprintf(stderr, "error: invalid value '%s' for '%s'\n%s", argv[a.i], a.flag.c_str(), polish_usage); return 2; };
    while (a.next()) {
        if (a.is("-r", "--reads")) reads = a.value();
        else if (a.is("-i", "--input")) in = a.value();
        else if (a.is("-o", "--out_dir")) out = a.value();
        else if (a.is("--kmer")) { k = (unsigned long)a.number(true); if (k < 11 || k > 31 || k % 2 == 0) return refuse(); }
        else if (a.is("--min_count")) { min_count = (unsigned long)a.number(true); if (min_count < 1 || min_count > 16383) return refuse(); has_min = true; }
        else if (a.is("--max_indel")) { max_indel = (unsigned long)a.number(true); if (max_indel < 1 || max_indel > 4) return refuse(); }
        else if (a.is("--rounds")) { rounds = (unsigned long)a.number(true); if (rounds < 1 || rounds > 10) return refuse(); }
        else if (a.is("--device")) device = atoi(a.value());
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (reads.empty() || in.empty() || out.empty()) return a.missing();
    const uint32_t t = (uint32_t)min_count;
    const int rc = ac_polish_fasta(reads.c_str(), in.c_str(), out.c_str(), (uint32_t)k, has_min ? &t : nullptr, (uint32_t)max_indel,
                                   (uint32_t)rounds, device, 1, nullptr);
    if (rc == AC_OK) {
        FILE* f = fopen((out + "/summary.tsv").c_str(), "rb");
        if (f) {
            char buf[1 << 16]; size_t n;
            while ((n = fread(buf, 1, sizeof buf, f)) > 0) fwrite(buf, 1, n, stdout);
            fclose(f);
        }
    }
    return finish(rc);
}

// `autocycler variants`: the alleles the reads carry beside the consensus, with every position's alternatives screened on the GPU (not in
// the reference).  summary.tsv also goes to stdout, byte for byte.
static const char* variants_usage =
    "Usage: autocycler variants --reads <READS> --input <FASTA> --out_dir <DIR> [--kmer 21] [--min_count N] [--max_indel 1]\n"
    "                           [--min_fraction 0.1] [--device N]\n\n"
    "Finds the alleles the reads carry beside the consensus, with every position's alternatives screened on the GPU: a substitution,\n"
    "or an insertion or deletion of up to --max_indel bases, whose k-mers the reads hold at least --min_count times, at a fraction of at\n"
    "least --min_fraction beside the consensus's own k-mers. This command is not in the reference. Writes variants.vcf (indels\n"
    "left-aligned) and summary.tsv (also to stdout).\n\n"
    "Options:\n"
    "  -r, --reads <READS>            Reads in FASTQ format, gzipped or not (required)\n"
    "  -i, --input <FASTA>            Assembly in FASTA format, gzipped or not (required)\n"
    "  -o, --out_dir <DIR>            Directory to create and write the VCF and summary into (required)\n"
    "      --kmer <KMER>              K-mer size, odd, 11 to 31 [default: 21]\n"
    "      --min_count <N>            Read count an alternative allele's k-mers need, 1 to 16383 [default: the valley of the reads'\n"
    "                                 k-mer spectrum]\n"
    "      --max_indel <L>            Longest insertion or deletion tried, 0 to 3 [default: 1]\n"
    "      --min_fraction <F>         Least alternative allele fraction, above 0 and at most 1 [default: 0.1]\n"
    "      --device <ORDINAL>         CUDA device [default: 0]\n";
static int variants_main(int argc, char** argv) {
    Args a{argc, argv, variants_usage};
    std::string reads, in, out; bool has_min = false;
    unsigned long k = 21, min_count = 0, max_indel = 1; double min_fraction = 0.1; int device = 0;
    auto refuse = [&]() { fprintf(stderr, "error: invalid value '%s' for '%s'\n%s", argv[a.i], a.flag.c_str(), variants_usage); return 2; };
    while (a.next()) {
        if (a.is("-r", "--reads")) reads = a.value();
        else if (a.is("-i", "--input")) in = a.value();
        else if (a.is("-o", "--out_dir")) out = a.value();
        else if (a.is("--kmer")) { k = (unsigned long)a.number(true); if (k < 11 || k > 31 || k % 2 == 0) return refuse(); }
        else if (a.is("--min_count")) { min_count = (unsigned long)a.number(true); if (min_count < 1 || min_count > 16383) return refuse(); has_min = true; }
        else if (a.is("--max_indel")) { max_indel = (unsigned long)a.number(true); if (max_indel > 3) return refuse(); }
        else if (a.is("--min_fraction")) { min_fraction = a.number(false); if (!(min_fraction > 0.0 && min_fraction <= 1.0)) return refuse(); }
        else if (a.is("--device")) device = atoi(a.value());
        else if (a.is("-h", "--help")) return a.help();
        else return a.unexpected();
    }
    if (reads.empty() || in.empty() || out.empty()) return a.missing();
    const uint32_t t = (uint32_t)min_count;
    const int rc = ac_variants_fasta(reads.c_str(), in.c_str(), out.c_str(), (uint32_t)k, has_min ? &t : nullptr, (uint32_t)max_indel,
                                     min_fraction, device, 1, nullptr);
    if (rc == AC_OK) {
        FILE* f = fopen((out + "/summary.tsv").c_str(), "rb");
        if (f) {
            char buf[1 << 16]; size_t n;
            while ((n = fread(buf, 1, sizeof buf, f)) > 0) fwrite(buf, 1, n, stdout);
            fclose(f);
        }
    }
    return finish(rc);
}

int main(int argc, char** argv) {
    if (argc >= 2 && strcmp(argv[1], "dotplot") == 0) return dotplot_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "resolve") == 0) return resolve_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "combine") == 0) return combine_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "decompress") == 0) return decompress_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "cluster") == 0) return cluster_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "trim") == 0) return trim_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "compress") == 0) return compress_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "clean") == 0) return clean_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "gfa2fasta") == 0) return gfa2fasta_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "table") == 0) return table_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "subsample") == 0) return subsample_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "helper") == 0) return helper_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "depth") == 0) return depth_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "qv") == 0) return qv_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "unassembled") == 0) return unassembled_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "polish") == 0) return polish_main(argc, argv);
    if (argc >= 2 && strcmp(argv[1], "variants") == 0) return variants_main(argc, argv);
    fprintf(stderr, "%s", compress_usage);
    return 2;
}
