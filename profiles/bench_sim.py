"""Measure whole failure scenarios through ClusterSimulation (rapid_b200/simulation.py) on one GPU:

    crash   N nodes, 1 % crashed (the Fig. 8 shape): ten quiet intervals, then one alerting interval and a fast-path view change
    churn   N nodes, 1 % crashed while 0.2 % join in the same windows
    leave   N nodes, 1 % leave gracefully (ClusterSimulation.leave): their observers raise the leave alerts in interval 0
    rolling N nodes (--churn-nodes), three waves of 1 % that leave and then rejoin with new NodeIds (a rolling restart)

leave and rolling run only when named; the default "both" is crash + churn.

Per scenario it reports the device time of a quiet and of an alerting interval (and the host clock of the first alerting one), every configuration's host-clock time split
into cut detection + tally, classic round, view change (cut lookup, applyCut, new configuration id) and handle re-creation,
and the whole scenario's wall time.  The scenario runs once to warm up, then --repeat times (default 1: one pass at 10⁶ nodes takes minutes);
the figures are the median.

    python profiles/bench_sim.py [--scenario crash|churn|leave|rolling|both] [--nodes 1000000] [--churn-nodes 100000] [--repeat 1]
                                 [--batch-order sender|shuffled|both] [--out FILE]

--check-windows NODES runs only the shuffled alerting interval at NODES nodes on a sweep handle and checks its first and last 256
receivers against the oracle's handlers (a few minutes of CPU at 10⁵ nodes: too long for a test).
--batch-order is ClusterSimulation's delivery model: "shuffled" gives every receiver its own batch order (sweep kernel), "both"
runs each scenario in both models in the same call.
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


def scenario(rb, W, n, n_joiners, seed, kind="crash", batch_order="sender"):
    s = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=seed, batch_order=batch_order)
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
            "first_alerting_interval": {k: first[0][k] for k in ("interval", "alerts", "cells", "leavers", "device_ms", "host_ms")} if first else None}


def window_check(rb, W, n, window=256, seed=0x5EED):
    """--check-windows: the alerting interval of `crash` at n nodes (1 % crashed, one batch per sender) on a sweep handle with
    shuffled batch order, and two `window`-receiver windows (the first and the last receivers) through the oracle's handlers, each
    walking its own order (tests/shuffled_ref.py): outputs, announced_in and proposal fingerprints must be equal"""
    import numpy as np
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from oracle import oracle_py as orc
    import shuffled_ref
    from helpers import OracleWorld
    K, H, L = 10, 9, 4
    w = OracleWorld(orc, n, K)
    view = rb.MembershipView.from_packed(K, *W.packed_endpoints(0, n))
    cfg = view.getCurrentConfigurationId(*W.node_ids(0, n))
    assert cfg == w.view.getCurrentConfigurationId()
    obs, ring0 = view.tables()[0], np.asarray(view.getRing(0))
    b = W.c2_simultaneous_crash(obs, n, 0.01, seed)
    order = np.argsort(b.src, kind="stable")
    src, dst, ring, st = b.src[order], b.dst[order], b.ring[order], b.status[order]
    off = np.append(np.unique(src, return_index=True)[1], len(src)).astype(np.int64)
    blocked = W.blocked_by_receiver(b.blocked, ring0, 0, n)
    cl = rb.VirtualCluster(view, H, L, kernel="sweep")
    t0 = time.perf_counter()
    res, ain = cl.handleBatches(cfg, src, dst, ring, st, off, blocked=blocked, batch_order_seed=seed)
    host_ms = (time.perf_counter() - t0) * 1e3
    dev_ms = cl.lastDeviceMs()[0]
    checked = []
    for base in (0, n - window):
        sim = orc.ClusterSim(w.view, K, H, L, window, receiver_base=base)
        t1 = time.perf_counter()
        o_len, o_ann, props, o_in = shuffled_ref.apply_batches(sim, src, dst, ring, st, cfg, off, blocked=blocked[base: base + window],
                                                               order_seed=seed, receiver_base=base)
        sl = slice(base, base + window)
        assert (res.proposal_len[sl] == o_len).all() and (res.announced[sl] == o_ann).all() and (ain[sl] == o_in).all(), base
        for r in np.nonzero(o_len)[0].tolist():
            assert (int(res.proposal_hash[base + r]), int(res.proposal_hash2[base + r])) == rb.proposal_fingerprint(props[r]), base + r
        checked.append({"receivers": [base, base + window], "announced": int((o_len > 0).sum()),
                        "oracle_s": time.perf_counter() - t1})
    cl.close()
    return {"check": "shuffled windows", "nodes": n, "batches": len(off) - 1, "cells": len(dst), "device_ms": dev_ms,
            "host_ms": host_ms, "windows": checked, "equal": True}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=1_000_000)
    ap.add_argument("--churn-nodes", type=int, default=100_000)
    ap.add_argument("--scenario", default="both", choices=["crash", "churn", "leave", "rolling", "both"])
    ap.add_argument("--repeat", type=int, default=1)
    ap.add_argument("--batch-order", default="sender", choices=["sender", "shuffled", "both"])
    ap.add_argument("--check-windows", type=int, default=0, metavar="NODES",
                    help="only the shuffled alerting interval at NODES nodes, checked against the oracle on two 256-receiver windows")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_sim.py measures the GPU; no CUDA device is visible")
    import rapid_b200 as rb
    from rapid_b200 import workloads as W
    card = gpu_card()
    lines = []
    if args.check_windows:
        res = dict(window_check(rb, W, args.check_windows), gpu=card)
        print(json.dumps(res), flush=True)
        lines.append(res)
        args.scenario = None
    orders = ["sender", "shuffled"] if args.batch_order == "both" else [args.batch_order]
    for (name, n, nj), order in ((x, o) for x in (("crash", args.nodes, 0), ("churn", args.churn_nodes, args.churn_nodes // 500),
                                                  ("leave", args.nodes, 0), ("rolling", args.churn_nodes, 0)) for o in orders):
        if args.scenario != name and not (args.scenario == "both" and name in ("crash", "churn")):
            continue
        kind = "crash" if name == "churn" else name
        scenario(rb, W, n, nj, 24, kind, order)                   # warm-up: module loads, allocations of every shape
        runs = [scenario(rb, W, n, nj, 24, kind, order) for _ in range(args.repeat)]
        med = lambda key: statistics.median(r[key] for r in runs)   # noqa: E731
        cfg_keys = ("detect_ms", "classic_ms", "view_change_ms", "handles_ms", "device_ms")
        cfgs = [dict(c, **{k: statistics.median(r["configurations"][i][k] for r in runs) for k in cfg_keys})
                for i, c in enumerate(runs[0]["configurations"])]
        gone = {"crash": "crashed", "churn": "crashed", "leave": "leavers", "rolling": "leavers_per_wave"}[name]
        res = {"scenario": name, "batch_order": order, "nodes": n, "joiners": nj, gone: n // 100, "gpu": card, "repeat": args.repeat,
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
