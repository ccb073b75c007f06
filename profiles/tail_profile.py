"""Per-kernel profile of the compress tail: every kernel and copy from the first unitig kernel (run_key, where finish() starts) through
the last GFA kernel and the copies that follow it, with the gap before each, for `ac_compress` on a BASELINE workload (cfg2 by default).
torch.profiler with CUDA activities, in a run of its own (tracing slows the host: end-to-end numbers come from bench.py).
usage: python profiles/tail_profile.py --out DIR [--workload cfg2] [--steps 5] [--warmup 3]
Writes DIR/tail_<workload>.json (every step's rows, the card's name and power limit) and prints one markdown table: per row the median
over the profiled steps."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def short_name(name):
    """ac_body_kernel<RunKeyBody>(...) -> RunKeyBody; memcpy rows keep their kind."""
    if "<" in name:
        inner = name[name.index("<") + 1:]
        depth, out = 1, []
        for ch in inner:
            depth += ch == "<"
            depth -= ch == ">"
            if depth == 0 or (depth == 1 and ch == ","):
                break
            out.append(ch)
        return "".join(out).strip()
    return name.split("(")[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2")
    ap.add_argument("--k", type=int, default=51)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from autocycler_b200 import api, synth
    if not torch.cuda.is_available():
        raise SystemExit("tail_profile.py: no CUDA device")
    gpu = bench.gpu_identity(0)
    assemblies = synth.make_assemblies(args.workload)
    stream = torch.cuda.Stream(device=0)
    torch.cuda.set_stream(stream)
    _, seqs, count = bench.prepare_sequences(assemblies, args.k)
    kg = api.KmerGraph(args.k, device=0, stream=stream.cuda_stream)
    kg.add_sequences(seqs, count, upload=False)
    kg.upload()
    for _ in range(args.warmup):
        api.UnitigGraph.compress(kg)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            api.UnitigGraph.compress(kg)
            torch.cuda.synchronize()
    events = []
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        start = e.time_range.start
        events.append((start, e.time_range.end, short_name(e.name)))
    events.sort()
    # one step's tail = from a RunKeyBody launch (finish() starts) through the last GFA kernel and the copies right after it (the text
    # to the host, the small counters); the next kernel belongs to the next step
    starts = [i for i, ev in enumerate(events) if ev[2] == "RunKeyBody"]
    steps = []
    for si, i0 in enumerate(starts):
        i1 = starts[si + 1] if si + 1 < len(starts) else len(events)
        seg = events[i0:i1]
        last = max(j for j, ev in enumerate(seg) if ev[2].startswith(("Gfa", "Path")))
        while last + 1 < len(seg) and seg[last + 1][2].startswith("Memcpy"):
            last += 1
        seg = seg[:last + 1]
        rows, prev_end = [], seg[0][0]
        for s, t, nm in seg:
            rows.append({"name": nm, "us": round(t - s, 2), "gap_us": round(s - prev_end, 2), "start_us": round(s - seg[0][0], 2)})
            prev_end = max(prev_end, t)
        steps.append({"rows": rows, "span_us": round(prev_end - seg[0][0], 2)})
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, f"tail_{args.workload}.json")
    json.dump({"gpu": gpu, "workload": args.workload, "k": args.k, "steps": steps}, open(path, "w"), indent=1)
    # the median step's table: rows line up across steps when every step launched the same kernels
    same = [st for st in steps if [r["name"] for r in st["rows"]] == [r["name"] for r in steps[0]["rows"]]]
    print(f"# {args.workload}, k={args.k}: {gpu['name']} at {gpu['power_limit_w']} W; {len(same)} of {len(steps)} steps alike; "
          f"tail span median {statistics.median(st['span_us'] for st in steps):.1f} us")
    print("| # | kernel / copy | us | gap before (us) | start (us) |")
    print("|---|---|---|---|---|")
    for j, r in enumerate(same[0]["rows"] if same else []):
        med = lambda key: statistics.median(st["rows"][j][key] for st in same)
        print(f"| {j} | {r['name']} | {med('us'):.1f} | {med('gap_us'):.1f} | {med('start_us'):.1f} |")
    print(f"wrote {path}")


if __name__ == "__main__":
    main()
