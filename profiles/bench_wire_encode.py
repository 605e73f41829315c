"""Timing of the wire-format egress (csrc/wire_encode.cu): the encode calls of two cases, each a host clock around a call that ends
in a stream synchronisation, median of --reps after one warm-up call, with the bytes the call wrote.

  interval : a C5-shaped failure-detector interval (--n nodes, 1 % crashed: about K * n / 100 alerts) -> one BatchedAlertMessage
             per sender, wrapped in RapidRequest
  votes    : every receiver of the same view announcing the cut of the crashed nodes -> n FastRoundPhase2bMessages sharing one body
  phase1b  : the n acceptors holding those votes answer one Phase1a -> n Phase1bMessages sharing one vval body

One JSON line per case on stdout, with the GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import rapid_b200 as rb  # noqa: E402
from rapid_b200 import _native as N  # noqa: E402
from rapid_b200 import workloads as W  # noqa: E402


def gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        return "unknown"


def timed(f, reps):
    f()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    n, K = a.n, 10
    hb, off, ports = W.packed_endpoints(0, n)
    view = rb.MembershipView.from_packed(K, hb, off, ports)
    view.setNodeIds(*W.node_ids(0, n))
    fd = rb.EdgeFailureDetectors(view, failure_threshold=1)
    flags = np.zeros(n, np.uint8)
    flags[np.random.default_rng(0).choice(n, n // 100, replace=False)] = rb.failure_detector.CRASHED
    fd.tick(flags, 1)
    alerts, cells = fd.tick(flags, 1)
    dec = rb.WireDecoder(view)
    card = gpu()

    med, lo, hi = timed(lambda: N.check(N.lib().rapid_wire_encode_alert_batches(dec._h, fd._h, N.WIRE_REQUEST, None, None)), a.reps)
    m, hbytes, nb, bbytes = dec.encodedCounts()
    print(json.dumps({"case": "interval", "n": n, "alerts": alerts, "messages": m, "bytes": hbytes + bbytes, "ms_median": med,
                      "ms_min": lo, "ms_max": hi, "gpu": card}), flush=True)

    vc = rb.VirtualCluster(view, 9, 4)
    src, dst, ring, status, cfg = fd.cells()
    vc.handleBatch(1, src, dst, ring, status, read_outputs=False)
    med, lo, hi = timed(lambda: N.check(N.lib().rapid_wire_encode_votes(dec._h, vc._h, 1, N.WIRE_REQUEST, None, None)), a.reps)
    m, hbytes, nb, bbytes = dec.encodedCounts()
    print(json.dumps({"case": "votes", "n": n, "messages": m, "bodies": nb, "body_bytes": bbytes, "header_bytes": hbytes,
                      "ms_median": med, "ms_min": lo, "ms_max": hi, "gpu": card}), flush=True)

    acc = rb.PaxosAcceptors(1, n)
    acc.registerFastRoundVotesFrom(vc)
    acc.handlePhase1aMessage((2, 1))
    med, lo, hi = timed(lambda: N.check(N.lib().rapid_wire_encode_phase1b(dec._h, acc._h, vc._h, N.WIRE_REQUEST, None, None)), a.reps)
    m, hbytes, nb, bbytes = dec.encodedCounts()
    print(json.dumps({"case": "phase1b", "n": n, "messages": m, "bodies": nb, "body_bytes": bbytes, "header_bytes": hbytes,
                      "ms_median": med, "ms_min": lo, "ms_max": hi, "gpu": card}), flush=True)


if __name__ == "__main__":
    main()
