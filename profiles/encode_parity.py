"""Digests of everything the wire encoder and the proposal census write on the benchmarked shapes, for comparing two builds
output for output, and the device memory the encoder holds.

  interval, votes, phase1b   the shapes of profiles/bench_wire_encode.py (--n nodes, 1 % crashed; one body)
  census one / thirty        the shapes of profiles/bench_census.py (C2, F = 100 crashed, one and thirty proposals)
  votes thirty               the fast-round votes of the thirty-proposal detector (thirty bodies)

Per encode: sha256 and length of the headers, header offsets, body ids, bodies, body offsets, sizes and senders.  Per census:
of every output array (classes, lists, statuses, in_cut against the decided cut, receiver classes).  encoder_bytes: the drop
in free device memory across the interval, votes and phase1b encodes of a fresh handle (cudaMemGetInfo, 2 MiB granules).
votes_thirty_ms: the thirty-body vote encode timed as bench_wire_encode.py times its calls (host clock around a call that ends in
a stream synchronisation, median of 20 after one warm-up), with the card's name and power limit.

    python profiles/encode_parity.py [--n 1000000] [--out FILE]"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

K, H, L, F, GROUPS = 10, 9, 4, 100, 30


def digest(**arrays):
    return {k: [len(a), hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()] for k, a in arrays.items()}


def encoded(dec):
    e = dec.encoded()
    return digest(headers=e.headers, header_off=e.header_off, body_ids=e.body_ids, bodies=e.bodies, body_off=e.body_off,
                  sizes=e.sizes(), senders=e.senders)


def census(cl, cut):
    c = cl.proposalCensus(cut)
    return digest(hash=c.hash, hash2=c.hash2, length=c.length, voters=c.voters, representative=c.representative, in_cut=c.in_cut,
                  list_off=c.list_off, ids=c.ids, status=c.status, classes=c.classes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("encode_parity.py runs the encoder on the GPU; no CUDA device is visible")
    import rapid_b200 as rb
    from rapid_b200 import _native as N
    from rapid_b200 import workloads as W
    n, res = args.n, {}

    # profiles/bench_wire_encode.py
    hb, off, ports = W.packed_endpoints(0, n)
    view = rb.MembershipView.from_packed(K, hb, off, ports)
    view.setNodeIds(*W.node_ids(0, n))
    fd = rb.EdgeFailureDetectors(view, failure_threshold=1)
    flags = np.zeros(n, np.uint8)
    flags[np.random.default_rng(0).choice(n, n // 100, replace=False)] = rb.failure_detector.CRASHED
    fd.tick(flags, 1)
    fd.tick(flags, 1)
    vc = rb.VirtualCluster(view, 9, 4)
    src, dst, ring, status, cfg = fd.cells()
    vc.handleBatch(1, src, dst, ring, status, read_outputs=False)
    acc = rb.PaxosAcceptors(1, n)
    acc.registerFastRoundVotesFrom(vc)
    acc.handlePhase1aMessage((2, 1))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    dec = rb.WireDecoder(view)
    dec.encodeAlertBatches(fd, as_request=True)
    res["interval"] = encoded(dec)
    dec.encodeVotes(vc, 1, as_request=True)
    res["votes"] = encoded(dec)
    dec.encodePhase1b(acc, vc, as_request=True)
    res["phase1b"] = encoded(dec)
    torch.cuda.synchronize()
    res["encoder_bytes"] = free0 - torch.cuda.mem_get_info()[0]
    for h in (dec, acc, vc, fd, view):
        h.close()

    # profiles/bench_census.py
    v = rb.MembershipView.from_packed(K, *W.packed_endpoints(0, n))
    obs, _ = v.tables()
    ring0 = np.asarray(v.getRing(0))
    b = W.c2_simultaneous_crash(obs, n, F / n, 5)
    blocked = W.blocked_by_receiver(b.blocked, ring0, 0, n)
    subjects = np.unique(b.dst)
    words = (n + 31) // 32
    r = np.arange(words * 32)
    rows = {}
    for g in range(GROUPS - 1):
        bits = (r % GROUPS == g).reshape(words, 32).astype(np.uint64)
        rows[int(subjects[g])] = ~(bits << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)
    bitmap = np.full((len(b.dst), words), 0xFFFFFFFF, np.uint32)
    for i, d in enumerate(b.dst.tolist()):
        if d in rows:
            bitmap[i] = rows[d]
    for name, bm in (("one", None), ("thirty", bitmap)):
        cl = rb.VirtualCluster(v, H, L, kernel="bucketed", max_subjects=len(subjects) + 64)
        cl.handleBatch(0, b.src, b.dst, b.ring, b.status, blocked=blocked, bitmap=bm, read_outputs=False)
        res["census_" + name] = census(cl, subjects)
        if name == "thirty":
            dec = rb.WireDecoder(v)
            dec.encodeVotes(cl, 1, as_request=True)
            res["votes_thirty"] = encoded(dec)
            res["votes_thirty_bodies"] = dec.encodedCounts()[2]
            ts = []
            for _ in range(21):
                t0 = time.perf_counter()
                N.check(N.lib().rapid_wire_encode_votes(dec._h, cl._h, 1, N.WIRE_REQUEST, None, None))
                ts.append((time.perf_counter() - t0) * 1e3)
            res["votes_thirty_ms"] = float(np.median(ts[1:]))
            res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                                        text=True).stdout.strip()
            dec.close()
        cl.close()
    print(json.dumps(res, sort_keys=True), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
