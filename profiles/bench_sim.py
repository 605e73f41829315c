"""Measure whole failure scenarios through ClusterSimulation (rapid_b200/simulation.py) on one GPU:

    crash   N nodes, 1 % crashed (the Fig. 8 shape): ten quiet intervals, then one alerting interval and a fast-path view change
    churn   N nodes, 1 % crashed while 0.2 % join in the same windows

Per scenario it reports the device time of a quiet and of an alerting interval, every configuration's host-clock time split
into cut detection + tally, classic round, view change (cut lookup, applyCut, new configuration id) and handle re-creation,
and the whole scenario's wall time.  The scenario runs once to warm up, then --repeat times (default 1: one pass at 10⁶ nodes takes minutes);
the figures are the median.

    python profiles/bench_sim.py [--scenario crash|churn|both] [--nodes 1000000] [--churn-nodes 100000] [--repeat 1] [--out FILE]
Prints one JSON object per scenario (and writes them to FILE)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def scenario(rb, W, n, n_joiners, seed):
    s = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=seed)
    crashed = W.pick_smallest(n, n // 100, seed)
    if n_joiners:
        hosts, ports = W.endpoints(n, n_joiners)
        s.addJoiners(hosts, ports, *W.node_ids(n, n_joiners))
    for t in crashed.tolist():
        s.setFlags(t, 1)
    t0 = time.perf_counter()
    out = s.run(15)
    wall = (time.perf_counter() - t0) * 1e3
    assert out["converged"], out
    quiet = [r["device_ms"] for r in s.intervals if r["event"] == "quiet"]
    alerting = [r["device_ms"] for r in s.intervals if r["event"] != "quiet"]
    cfgs = [{k: h[k] for k in ("path", "intervals", "size_before", "size", "announced", "detect_ms", "classic_ms", "view_change_ms",
                               "handles_ms", "device_ms")} for h in s.history]
    s.close()
    print("%s nodes: %.0f ms" % (n, wall), file=sys.stderr, flush=True)
    return {"wall_ms": wall, "quiet_interval_device_ms": min(quiet) if quiet else None,
            "alerting_interval_device_ms": max(alerting) if alerting else None, "configurations": cfgs, "cut": len(crashed) + n_joiners}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=1_000_000)
    ap.add_argument("--churn-nodes", type=int, default=100_000)
    ap.add_argument("--scenario", default="both", choices=["crash", "churn", "both"])
    ap.add_argument("--repeat", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_sim.py measures the GPU; no CUDA device is visible")
    import rapid_b200 as rb
    from rapid_b200 import workloads as W
    card = gpu_card()
    lines = []
    for name, n, nj in (("crash", args.nodes, 0), ("churn", args.churn_nodes, args.churn_nodes // 500)):
        if args.scenario not in (name, "both"):
            continue
        scenario(rb, W, n, nj, 24)                                # warm-up: module loads, allocations of every shape
        runs = [scenario(rb, W, n, nj, 24) for _ in range(args.repeat)]
        med = lambda key: statistics.median(r[key] for r in runs)   # noqa: E731
        cfg_keys = ("detect_ms", "classic_ms", "view_change_ms", "handles_ms", "device_ms")
        cfgs = [dict(c, **{k: statistics.median(r["configurations"][i][k] for r in runs) for k in cfg_keys})
                for i, c in enumerate(runs[0]["configurations"])]
        res = {"scenario": name, "nodes": n, "joiners": nj, "crashed": n // 100, "gpu": card, "repeat": args.repeat,
               "wall_ms_median": med("wall_ms"), "wall_ms_all": [r["wall_ms"] for r in runs],
               "quiet_interval_device_ms": med("quiet_interval_device_ms"),
               "alerting_interval_device_ms": med("alerting_interval_device_ms"), "configurations": cfgs,
               "note": "device_ms: CUDA events of the detector tick, the batch handling and the tally (and classic phases); "
                       "*_ms of a configuration: host clock around calls that end in a device synchronise"}
        print(json.dumps(res), flush=True)
        lines.append(res)
    if args.out:
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
