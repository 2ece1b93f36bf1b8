"""Turn timeline of a two-thread search: where the tree stream and the network stream wait for each other.

Runs searches of a bench.py workload (default: the headline, Threads 2) under torch.profiler with CUDA activities, in a
run of its own, and reads the kernels of both streams back from the trace.  The tree stream is the one the select
kernel runs on; every other stream (the network stream and its value-head branch) counts as the network.  A turn
starts at an update_kernel, or at a select kernel when the turn so far has one already (the first two turns of a
search have no update); the root phase of a search is left out.  Per turn the JSON lists
  - every kernel of both streams in the turn's window, start and end in microseconds from the search's root_kernel;
  - for each tree-stream kernel, the time from its predecessor's end to its own start (`gap_us`), and how much of that
    gap a tower kernel (rise_trunk*) was running (`gap_beside_tower_us`);
  - the stretches of the window in which no network kernel runs (`net_idle`, and their sum `net_idle_us`).
The summary averages them over all profiled turns.

    python tools/prof_turn.py --out DIR [--label NAME] [--config M|2|3] [--searches 2] [--warmup 3]

ARA_B200_LIB selects another build of the library, e.g. that of an earlier commit, for a before / after pair.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def short(name):
    """kernel name without return type, namespace, template arguments and parameter list"""
    n = name[5:] if name.startswith("void ") else name
    return n.split("(")[0].split("<")[0].replace("ara::", "")


def kernels_from_trace(path):
    ev = json.load(open(path))
    ev = ev["traceEvents"] if isinstance(ev, dict) else ev
    ks = [e for e in ev if e.get("cat") == "kernel" and e.get("ph") == "X"]
    out = [{"name": short(e["name"]), "full": e["name"], "stream": e.get("args", {}).get("stream"),
            "start": float(e["ts"]), "end": float(e["ts"]) + float(e["dur"])} for e in ks]
    out.sort(key=lambda k: k["start"])
    return out


def union_len(intervals, lo, hi):
    """length of the union of `intervals` clipped to [lo, hi), and the uncovered stretches"""
    iv = sorted((max(a, lo), min(b, hi)) for a, b in intervals if b > lo and a < hi)
    covered, holes, cur = 0.0, [], lo
    for a, b in iv:
        if a > cur:
            holes.append((cur, a))
        if b > cur:
            covered += b - max(a, cur)
            cur = b
    if cur < hi:
        holes.append((cur, hi))
    return covered, holes


def analyse(kernels):
    selects = [k for k in kernels if k["name"].startswith("select")]
    if not selects:
        raise SystemExit("no select kernel in the trace")
    streams = {}
    for k in selects:
        streams[k["stream"]] = streams.get(k["stream"], 0) + 1
    tree_stream = max(streams, key=streams.get)
    tree = [k for k in kernels if k["stream"] == tree_stream]
    net = [k for k in kernels if k["stream"] != tree_stream]
    towers = [(k["start"], k["end"]) for k in net if k["name"].startswith("rise_trunk")]
    # searches: each begins at a root_kernel on the tree stream
    roots = [i for i, k in enumerate(tree) if k["name"] == "root_kernel"]
    searches = []
    for si, r0 in enumerate(roots):
        r1 = roots[si + 1] if si + 1 < len(roots) else len(tree)
        seq = tree[r0:r1]
        t0 = seq[0]["start"]
        turns, cur, has_select = [], None, False
        for i, k in enumerate(seq):
            select = k["name"].startswith("select")
            if k["name"] == "update_kernel" or (select and (cur is None or has_select)):
                if cur:
                    turns.append(cur)
                cur, has_select = [], False
            has_select = has_select or select
            if cur is not None:
                cur.append((i, k))
        if cur:
            turns.append(cur)
        out_turns = []
        for ti, turn in enumerate(turns):
            lo = turn[0][1]["start"]
            hi = turns[ti + 1][0][1]["start"] if ti + 1 < len(turns) else turn[-1][1]["end"]
            tk = []
            for i, k in turn:
                prev_end = seq[i - 1]["end"] if i > 0 else k["start"]
                gap = max(0.0, k["start"] - prev_end)
                beside, _ = union_len(towers, prev_end, k["start"]) if gap > 0 else (0.0, [])
                tk.append({"name": k["name"], "start_us": k["start"] - t0, "end_us": k["end"] - t0, "gap_us": gap,
                           "gap_beside_tower_us": beside})
            nk = [{"name": k["name"], "stream": k["stream"], "start_us": k["start"] - t0, "end_us": k["end"] - t0}
                  for k in net if k["end"] > lo and k["start"] < hi]
            busy, holes = union_len([(k["start"], k["end"]) for k in net], lo, hi)
            out_turns.append({"turn": ti, "start_us": lo - t0, "end_us": hi - t0, "tree": tk, "net": nk,
                              "net_idle_us": (hi - lo) - busy,
                              "net_idle": [[a - t0, b - t0] for a, b in holes if b - a > 0.5]})
        searches.append({"search": si, "span_us": seq[-1]["end"] - t0, "turns": out_turns})
    return tree_stream, searches


def summarise(searches):
    per_kernel, n_turns, idle, length = {}, 0, 0.0, 0.0
    for s in searches:
        for t in s["turns"]:
            n_turns += 1
            idle += t["net_idle_us"]
            length += t["end_us"] - t["start_us"]
            for k in t["tree"]:
                d = per_kernel.setdefault(k["name"], {"count": 0, "dur_us": 0.0, "gap_us": 0.0, "gap_beside_tower_us": 0.0})
                d["count"] += 1
                d["dur_us"] += k["end_us"] - k["start_us"]
                d["gap_us"] += k["gap_us"]
                d["gap_beside_tower_us"] += k["gap_beside_tower_us"]
    for d in per_kernel.values():
        for f in ("dur_us", "gap_us", "gap_beside_tower_us"):
            d[f] /= d["count"]
    return {"turns": n_turns, "mean_turn_us": length / max(1, n_turns), "mean_net_idle_per_turn_us": idle / max(1, n_turns),
            "mean_search_us": sum(s["span_us"] for s in searches) / max(1, len(searches)), "tree_kernels": per_kernel}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory (turns_<label>.json and the raw trace)")
    ap.add_argument("--label", default="run")
    ap.add_argument("--config", default="M", choices=["M", "2", "3"])
    ap.add_argument("--searches", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("prof_turn.py needs a CUDA device")
    from torch.profiler import ProfilerActivity, profile

    import bench
    from crazyara_b200 import synthetic
    from crazyara_b200.engine import BoardState, MCTSAgent, default_settings
    from crazyara_b200.nn import NeuralNetAPI
    from crazyara_b200.weights import export_blob

    variant, vid, mode, family, cin, pch, version, batch, sims = bench.WORKLOADS[args.config]
    arch = bench.make_arch(family, cin, pch)
    os.makedirs(args.out, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        blob = export_blob(synthetic.random_state_dict(arch, 0), arch, os.path.join(tmp, "net.arab"), input_version=version * 10)
        net = NeuralNetAPI("gpu", 0, batch, blob)
        agent = MCTSAgent(net, default_settings(mode, batch_size=batch, simulations=sims, threads=2, input_version=version), 0, 1)
        for _ in range(args.warmup):
            agent.evaluate_board_state(BoardState().set("", False, vid))
        torch.cuda.synchronize()
        trace = os.path.join(args.out, f"trace_{args.label}.json")
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.searches):
                agent.evaluate_board_state(BoardState().set("", False, vid))
            torch.cuda.synchronize()
        prof.export_chrome_trace(trace)
        agent.close()
        net.close()
    tree_stream, searches = analyse(kernels_from_trace(trace))
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        card = torch.cuda.get_device_name(0)
    summary = summarise(searches)
    res = {"label": args.label, "config": args.config, "card": card, "tree_stream": tree_stream, "summary": summary,
           "searches": searches}
    path = os.path.join(args.out, f"turns_{args.label}.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"label": args.label, "card": card, **{k: v for k, v in summary.items()}}))


if __name__ == "__main__":
    main()
