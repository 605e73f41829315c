"""Time the proposal census (rapid_cd_proposal_census + rapid_cd_read_census) at 10^6 receivers against the host path it
replaces: readOutputs (21 B per receiver to the host), grouping the announcers' fingerprints on the host (numpy), and one
rapid_cd_get_proposal per distinct proposal.

Two shapes, both on a bucketed handle over a view of 10^6 members, F = 100 crashed (C2, crashed receivers blocked), one batch:
  one      every live receiver gets every cell: one proposal
  thirty   receivers split into 30 groups by r mod 30; group g < 29 is not delivered the cells about the g-th crashed node
           (RAPID_DELIVERY_BITMAP), so it announces the cut without that node: 30 proposals
Each side is timed by the host clock around the whole call, which ends in a device synchronisation (both return their results
to the host), median of --reps after --warmup; the two results are checked equal first.

    python profiles/bench_census.py [--n 1000000] [--reps 20] [--warmup 3] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

K, H, L, F, GROUPS = 10, 9, 4, 100, 30


def gpu_card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def census(N, cl):
    """device path: the census, then every class's fingerprint, voters, representative and list to the host"""
    nc, ne = C.c_int64(0), C.c_int64(0)
    N.check(N.lib().rapid_cd_proposal_census(cl._h, None, 0, C.byref(nc), C.byref(ne)))
    h1, h2 = np.zeros(nc.value, np.uint64), np.zeros(nc.value, np.uint64)
    ln, vo, rep = (np.zeros(nc.value, np.int32) for _ in range(3))
    off, ids = np.zeros(nc.value + 1, np.int64), np.zeros(ne.value, np.int32)
    N.check(N.lib().rapid_cd_read_census(cl._h, N.ptr(h1), N.ptr(h2), N.ptr(ln), N.ptr(vo), N.ptr(rep), None, N.ptr(off), N.ptr(ids), None))
    return [(int(h1[i]), int(h2[i]), int(vo[i]), int(rep[i]), ids[off[i]: off[i + 1]].tolist()) for i in range(nc.value)]


def host_path(cl):
    """readOutputs, fingerprints grouped on the host, one getProposal per distinct proposal"""
    out = cl.readOutputs()
    now = np.nonzero(out.proposal_len > 0)[0]
    key = np.stack([out.proposal_hash[now], out.proposal_hash2[now], out.proposal_len[now].astype(np.uint64)], axis=1)
    u, first, counts = np.unique(key, axis=0, return_index=True, return_counts=True)
    order = np.argsort(now[first], kind="stable")                  # classes in order of their lowest receiver
    return [(int(u[j, 0]), int(u[j, 1]), int(counts[j]), int(now[first[j]]), cl.getProposal(int(now[first[j]]))) for j in order]


def median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_census.py measures the GPU; no CUDA device is visible")
    import rapid_b200 as rb
    from rapid_b200 import _native as N
    from rapid_b200 import workloads as W
    n = args.n
    v = rb.MembershipView.from_packed(K, *W.packed_endpoints(0, n))
    obs, _ = v.tables()
    ring0 = np.asarray(v.getRing(0))
    b = W.c2_simultaneous_crash(obs, n, F / n, 5)
    blocked = W.blocked_by_receiver(b.blocked, ring0, 0, n)
    subjects = np.unique(b.dst)
    words = (n + 31) // 32
    r = np.arange(words * 32)
    rows = {}
    for g in range(GROUPS - 1):                                    # the receivers of group g, as bitmap words
        bits = (r % GROUPS == g).reshape(words, 32).astype(np.uint64)
        rows[int(subjects[g])] = ~(bits << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)
    bitmap = np.full((len(b.dst), words), 0xFFFFFFFF, np.uint32)
    for i, d in enumerate(b.dst.tolist()):
        if d in rows:
            bitmap[i] = rows[d]
    res = {"bench": "proposal_census", "receivers": n, "crashed": int(len(subjects)), "gpu": gpu_card(), "reps": args.reps,
           "timing": "host clock around each call, which ends in a device synchronisation; median (min, max) ms", "shapes": []}
    for name, bm in (("one", None), ("thirty", bitmap)):
        cl = rb.VirtualCluster(v, H, L, kernel="bucketed", max_subjects=len(subjects) + 64)
        cl.handleBatch(0, b.src, b.dst, b.ring, b.status, blocked=blocked, bitmap=bm, read_outputs=False)
        a, h = census(N, cl), host_path(cl)
        assert a == h, name
        c_ms = median_ms(lambda: census(N, cl), args.reps, args.warmup)
        h_ms = median_ms(lambda: host_path(cl), args.reps, args.warmup)
        row = {"shape": name, "classes": len(a), "announcers": int(sum(x[2] for x in a)), "entries": int(sum(len(x[4]) for x in a)),
               "census_ms": c_ms, "host_path_ms": h_ms, "speedup": h_ms[0] / c_ms[0]}
        print("%-6s classes %3d  census %.3f ms  host path %.3f ms  (x%.1f)" % (name, len(a), c_ms[0], h_ms[0], row["speedup"]),
              file=sys.stderr, flush=True)
        res["shapes"].append(row)
        cl.close()
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
