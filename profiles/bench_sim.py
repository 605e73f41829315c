"""Measure whole failure scenarios through ClusterSimulation (rapid_b200/simulation.py) on one GPU:

    crash   N nodes, 1 % crashed (the Fig. 8 shape): ten quiet intervals, then one alerting interval and a fast-path view change
    churn   N nodes, 1 % crashed while 0.2 % join in the same windows
    leave   N nodes, 1 % leave gracefully (ClusterSimulation.leave): their observers raise the leave alerts in interval 0
    rolling N nodes (--churn-nodes), three waves of 1 % that leave and then rejoin with new NodeIds (a rolling restart)

leave and rolling run only when named; the default "both" is crash + churn.

Per scenario it reports the device time of a quiet and of an alerting interval, every configuration's host-clock time split
into cut detection + tally, classic round, view change (cut lookup, applyCut, new configuration id) and handle re-creation,
and the whole scenario's wall time.  The scenario runs once to warm up, then --repeat times (default 1: one pass at 10⁶ nodes takes minutes);
the figures are the median.

    python profiles/bench_sim.py [--scenario crash|churn|leave|rolling|both] [--nodes 1000000] [--churn-nodes 100000] [--repeat 1]
                                 [--out FILE]
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


def scenario(rb, W, n, n_joiners, seed, kind="crash"):
    s = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=seed)
    crashed = W.pick_smallest(n, (3 if kind == "rolling" else 1) * (n // 100), seed)
    if n_joiners:
        hosts, ports = W.endpoints(n, n_joiners)
        s.addJoiners(hosts, ports, *W.node_ids(n, n_joiners))
    t0 = time.perf_counter()
    if kind == "crash":
        for t in crashed.tolist():
            s.setFlags(t, 1)
        out = s.run(15)
    elif kind == "leave":
        s.leave(crashed.tolist())
        out = s.run(15)
    else:                                                         # rolling: each wave leaves, then rejoins with new NodeIds
        for k in range(3):
            wave = crashed[k::3].tolist()
            s.leave(wave)
            out = s.run(15)
            assert out["converged"], out
            hi, lo = W.node_ids((1 << 40) + k * len(wave), len(wave))
            for j, t in enumerate(wave):
                s.rejoin(t, int(hi[j]), int(lo[j]))
            out = s.run(15)
    wall = (time.perf_counter() - t0) * 1e3
    assert out["converged"], out
    first = [r for r in s.intervals if r["event"] != "quiet"][:1]
    quiet = [r["device_ms"] for r in s.intervals if r["event"] == "quiet"]
    alerting = [r["device_ms"] for r in s.intervals if r["event"] != "quiet"]
    cfgs = [{k: h[k] for k in ("path", "intervals", "size_before", "size", "announced", "detect_ms", "classic_ms", "view_change_ms",
                               "handles_ms", "device_ms")} for h in s.history]
    s.close()
    print("%s nodes: %.0f ms" % (n, wall), file=sys.stderr, flush=True)
    return {"wall_ms": wall, "quiet_interval_device_ms": min(quiet) if quiet else None,
            "alerting_interval_device_ms": max(alerting) if alerting else None, "configurations": cfgs, "cut": len(crashed) + n_joiners,
            "intervals_to_first_decision": sum(c["intervals"] for c in cfgs[:1]),
            "first_alerting_interval": {k: first[0][k] for k in ("interval", "alerts", "cells", "leavers", "device_ms")} if first else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=1_000_000)
    ap.add_argument("--churn-nodes", type=int, default=100_000)
    ap.add_argument("--scenario", default="both", choices=["crash", "churn", "leave", "rolling", "both"])
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
    for name, n, nj in (("crash", args.nodes, 0), ("churn", args.churn_nodes, args.churn_nodes // 500), ("leave", args.nodes, 0),
                        ("rolling", args.churn_nodes, 0)):
        if args.scenario != name and not (args.scenario == "both" and name in ("crash", "churn")):
            continue
        kind = "crash" if name == "churn" else name
        scenario(rb, W, n, nj, 24, kind)                          # warm-up: module loads, allocations of every shape
        runs = [scenario(rb, W, n, nj, 24, kind) for _ in range(args.repeat)]
        med = lambda key: statistics.median(r[key] for r in runs)   # noqa: E731
        cfg_keys = ("detect_ms", "classic_ms", "view_change_ms", "handles_ms", "device_ms")
        cfgs = [dict(c, **{k: statistics.median(r["configurations"][i][k] for r in runs) for k in cfg_keys})
                for i, c in enumerate(runs[0]["configurations"])]
        gone = {"crash": "crashed", "churn": "crashed", "leave": "leavers", "rolling": "leavers_per_wave"}[name]
        res = {"scenario": name, "nodes": n, "joiners": nj, gone: n // 100, "gpu": card, "repeat": args.repeat,
               "intervals_to_first_decision": runs[0]["intervals_to_first_decision"],
               "first_alerting_interval": runs[0]["first_alerting_interval"],
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
