"""The insert kernel's register budget, swept: builds libautocycler_gpu.so with the insert compiled for each number of resident 256-thread
CTAs per SM (`-DAC_INSERT_CTAS=n`: 64 / 85 / 128 registers at 4 / 3 / 2), prints ptxas's registers, stack and spill bytes of every
`InsertBody` and `AdjacencyBody` instantiation, then times `insert_kernel` (CUDA events around its launch) on a workload, the builds
alternated round by round, each run in a process of its own, every GFA checked against the oracle's committed SHA-256.

  python profiles/insert_budget_sweep.py [--ctas 4 3 2] [--rounds 4] [--lib NAME=PATH ...] [--out DIR] [--build-only]

Builds go to --out (default: a temporary directory).  `--lib` adds a library built elsewhere (another commit's) to the alternation.
Needs `make -C autocycler_b200/csrc` first: the host objects are linked from its build directory."""
import argparse
import glob
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "autocycler_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVFLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC,-O3"]


def build(ctas, out):
    """-> (library path, {kernel: (registers, stack bytes, spill store bytes, spill load bytes)}) for InsertBody / AdjacencyBody."""
    d = os.path.join(out, f"ctas{ctas}")
    os.makedirs(d, exist_ok=True)
    obj = os.path.join(d, "pipeline.o")
    r = subprocess.run([NVCC, *NVFLAGS, f"-DAC_INSERT_CTAS={ctas}", "-Xptxas", "-v", "-c", os.path.join(CSRC, "pipeline.cu"), "-o", obj],
                       check=True, capture_output=True, text=True)
    host = sorted(o for o in glob.glob(os.path.join(CSRC, "build", "*.o")) if not o.endswith("pipeline.o"))
    if not host:
        raise SystemExit("no host objects: run `make -C autocycler_b200/csrc` first")
    lib = os.path.join(d, "libautocycler_gpu.so")
    subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", lib, obj, *host, "-lz", "-Xlinker", "-z,defs", "-lpthread"], check=True)
    return lib, ptxas_table(r.stderr)


def ptxas_table(log):
    rows, name = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
            continue
        if name is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            stack = tuple(int(x) for x in m.groups())
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m:
            pretty = subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip()
            b = re.search(r"(InsertBody|AdjacencyBody)<(\d+)>", pretty)
            if b and "ac_body_kernel" in pretty:
                rows[f"{b.group(1)}<{b.group(2)}>"] = (int(m.group(1)), *stack)
            name = None
    return rows


def time_one(lib, workload, k, steps, warmup):
    """One process, one library: `steps` builds after `warmup`, insert_kernel of each, and the GFA's SHA-256 against the golden."""
    sys.path.insert(0, ROOT)
    import torch
    from autocycler_b200 import api, synth
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "config_goldens.json")))
    with tempfile.TemporaryDirectory() as d:
        synth.write_assemblies(synth.make_assemblies(workload), d)
        kg, _, _ = api.load_sequences(d, k, lib=api.load_library(lib))
    want = golden[f"{workload}_k{k}"]["sha256"]
    ins, ok = [], True
    for i in range(warmup + steps):
        kg.upload()
        g = api.UnitigGraph.compress(kg)
        torch.cuda.synchronize()
        if i >= warmup:
            ins.append(g.timings().insert_kernel)
            ok = ok and hashlib.sha256(bytes(g.gfa_view())).hexdigest() == want
    ins.sort()
    print(json.dumps({"insert_kernel_ms_median": round(ins[len(ins) // 2], 3), "min": round(ins[0], 3), "max": round(ins[-1], 3), "parity": ok}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ctas", type=int, nargs="*", default=[4, 3, 2])
    ap.add_argument("--lib", action="append", default=[], help="NAME=PATH of another build to time alongside")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--workload", default="cfg2")
    ap.add_argument("--k", type=int, default=51)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--time-one", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.time_one:
        time_one(args.time_one, args.workload, args.k, args.steps, args.warmup)
        return
    out = args.out or tempfile.mkdtemp(prefix="insert_sweep_")
    libs = dict(x.split("=", 1) for x in args.lib)
    for n in args.ctas:
        lib, regs = build(n, out)
        libs[f"ctas{n}"] = lib
        for kern, (r, stack, st, ld) in sorted(regs.items()):
            print(f"ctas={n} {kern}: {r} registers, {stack} B stack, {st} B spill stores, {ld} B spill loads", flush=True)
    if args.build_only:
        return
    results = {name: [] for name in libs}
    for rnd in range(args.rounds):
        for name, lib in libs.items():
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--time-one", lib, "--workload", args.workload, "--k", str(args.k),
                                "--steps", str(args.steps), "--warmup", str(args.warmup)], check=True, capture_output=True, text=True)
            res = json.loads(r.stdout.strip().splitlines()[-1])
            results[name].append(res)
            print(f"round {rnd} {name}: {json.dumps(res)}", flush=True)
    for name, rs in results.items():
        med = sorted(r["insert_kernel_ms_median"] for r in rs)
        print(f"{name}: insert_kernel {med[0]:.3f}-{med[-1]:.3f} ms over {len(rs)} runs, parity {all(r['parity'] for r in rs)}")


if __name__ == "__main__":
    main()
