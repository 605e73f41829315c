"""The K/H/L sensitivity study of the Rapid paper (§6, Fig. 11: 1000 processes, F crashed, alerts delivered to each process in
uniform random order, conflict rate vs H - L) on the device's shuffled batch delivery (RAPID_DELIVERY_SHUFFLED_BATCHES).

Grid: N = 1000; F in {2, 4, 8, 16} crashed nodes (workloads.pick_smallest per repetition seed); (K, H, L) in {(10, 9, 3),
(10, 9, 4), (10, 8, 3), (10, 8, 2), (10, 7, 3)}; --reps repetitions per cell (default 20).  In a repetition every live
observer's DOWN alert about a crashed node is its own batch, the N - F live nodes receive the batches each in its own order
(one sweep VirtualCluster, crashed receivers blocked), and one FastPaxos tally counts the announced proposals.  Per cell:
the fraction of repetitions with >= 2 distinct announced proposals ("conflict"), the fraction without a fast quorum, and the
mean number of distinct proposals.

    python profiles/conflict_study.py [--reps 20] [--oracle] [--out FILE]

--oracle runs the same grid on the CPU through the oracle's literal handlers (tests/shuffled_ref.py); the outcomes are
deterministic, so both runs print the same table.  The paper's timing model (when alerts are generated and sent) is not
reproduced: the figures are context, not a reproduction."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

N = 1000
FS = (2, 4, 8, 16)
KHL = ((10, 9, 3), (10, 9, 4), (10, 8, 3), (10, 8, 2), (10, 7, 3))


def gpu_card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def repetition(W, obs, F, rep):
    """-> (seed, crashed ids, src, dst, ring, status, batch_off): one batch per (observer, subject) alert, observers ascending"""
    seed = 7919 * F + rep
    crashed = W.pick_smallest(N, F, seed)
    c = W.crash_cells(obs, crashed, N)
    order = np.lexsort((c["ring"], c["dst"], c["src"]))
    src, dst, ring, st = (c[k][order] for k in ("src", "dst", "ring", "status"))
    key = src.astype(np.int64) * N + dst
    first = np.nonzero(np.r_[True, key[1:] != key[:-1]])[0]
    return seed, crashed, src, dst, ring, st, np.append(first, len(src)).astype(np.int64)


def device_cell(rb, W, view, obs, ring0, cfg, K, H, L, F, reps):
    out = []
    for rep in range(reps):
        seed, crashed, src, dst, ring, st, off = repetition(W, obs, F, rep)
        dead = np.zeros(N, np.uint8)
        dead[crashed] = 1
        blocked = W.blocked_by_receiver(dead, ring0, 0, N)
        cl = rb.VirtualCluster(view, H, L, kernel="sweep")
        res, _ = cl.handleBatches(cfg, src, dst, ring, st, off, blocked=blocked, batch_order_seed=seed)
        now = res.proposal_len > 0
        distinct = len(set(zip(res.proposal_hash[now].tolist(), res.proposal_hash2[now].tolist(), res.proposal_len[now].tolist())))
        fp = rb.FastPaxos(cfg, N)
        decided = fp.tallyCluster(cl).decided
        fp.close()
        cl.close()
        out.append((distinct, decided))
    return out


def oracle_cell(orc, S, W, ow, obs, ring0, cfg, K, H, L, F, reps):
    out = []
    for rep in range(reps):
        seed, crashed, src, dst, ring, st, off = repetition(W, obs, F, rep)
        dead = np.zeros(N, np.uint8)
        dead[crashed] = 1
        blocked = dead[ring0]
        sim = orc.ClusterSim(ow.view, K, H, L, N)
        o_len, _, props, _ = S.apply_batches(sim, src, dst, ring, st, cfg, off, blocked=blocked, order_seed=seed)
        tally = orc.FastPaxosTally(ow.u, cfg, N)
        decided = False
        for r in np.nonzero(o_len)[0].tolist():
            decided |= tally.handleFastRoundProposal(int(ring0[r]), cfg, props[r])
        out.append((len({tuple(sorted(p)) for p in props if p}), bool(tally.decided() or decided)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--oracle", action="store_true", help="run the grid on the CPU through the oracle")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from rapid_b200 import workloads as W
    table = []
    if args.oracle:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from oracle import oracle_py as orc
        import shuffled_ref as S
        from helpers import OracleWorld
        orc.build()
        card = "cpu (oracle)"
    else:
        import torch
        if not torch.cuda.is_available():
            raise SystemExit("conflict_study.py runs on the GPU (or --oracle on the CPU); no CUDA device is visible")
        import rapid_b200 as rb
        card = gpu_card()
        hb, ho, ports = W.packed_endpoints(0, N)
    for K, H, L in KHL:
        if args.oracle:
            ow = OracleWorld(orc, N, K)
            obs, ring0, cfg = ow.tables()[0], ow.ring0(), ow.view.getCurrentConfigurationId()
        else:
            view = rb.MembershipView.from_packed(K, hb, ho, ports)
            hi, lo = W.node_ids(0, N)
            cfg = view.getCurrentConfigurationId(hi, lo)
            obs, ring0 = view.tables()[0], np.asarray(view.getRing(0))
        for F in FS:
            runs = (oracle_cell(orc, S, W, ow, obs, ring0, cfg, K, H, L, F, args.reps) if args.oracle
                    else device_cell(rb, W, view, obs, ring0, cfg, K, H, L, F, args.reps))
            d = np.array([r[0] for r in runs])
            row = {"K": K, "H": H, "L": L, "H-L": H - L, "F": F, "reps": args.reps,
                   "conflict": float((d >= 2).mean()), "no_fast_quorum": float(np.mean([not r[1] for r in runs])),
                   "mean_distinct": float(d.mean())}
            print("K=%d H=%d L=%d F=%2d  conflict %.3f  no fast quorum %.3f  distinct %.2f"
                  % (K, H, L, F, row["conflict"], row["no_fast_quorum"], row["mean_distinct"]), file=sys.stderr, flush=True)
            table.append(row)
    res = {"study": "conflict", "nodes": N, "gpu": card, "table": table}
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
