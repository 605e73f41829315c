"""Per-process agreement on conflict_study.py's grid (the Rapid paper's §6 / Fig. 11 setting: 1000 processes, F crashed, alerts
delivered to each process in its own order), from the device's proposal census (VirtualCluster.proposalCensus).

Same grid and repetitions as conflict_study.py (its N, FS, KHL and repetition()).  Per repetition the census groups the
announcers by proposal; the majority is the most-voted proposal (ties: the one with the lowest announcing receiver), every other
one a minority, measured against the majority by a second census with cut = the majority's ids.  Per cell:

* disagree       mean over repetitions of the share of announcers whose proposal is not the majority's — a per-process
                 conflict rate, the closer analogue of the paper's figure than conflict_study.py's "any conflict" fraction;
* subset         over the repetitions with a minority, the fraction in which every minority proposal is a strict subset of
                 the majority's (null when no repetition had one);
* missing/extra  mean over all minority proposals of the cell of |majority - minority| and |minority - majority| (null likewise).

    python profiles/conflict_census.py [--reps 20] [--oracle] [--out FILE]

--oracle computes the same from the oracle's per-receiver proposals (tests/shuffled_ref.py) on the CPU; the outcomes are
deterministic, so both runs print the same table."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import numpy as np  # noqa: E402

from conflict_study import FS, KHL, N, gpu_card, repetition  # noqa: E402


def summarize(rep_classes):
    """rep_classes: per repetition, [(voters, frozenset of ids)] in order of lowest announcing receiver -> (disagree, subset flag or
    None, [(missing, extra)] of the minorities)"""
    if not rep_classes:
        return 0.0, None, []
    voters = np.array([v for v, _ in rep_classes])
    m = int(np.argmax(voters))                              # first maximum: the lowest representative
    maj = rep_classes[m][1]
    minor = [ids for i, (_, ids) in enumerate(rep_classes) if i != m]
    dist = [(len(maj - ids), len(ids - maj)) for ids in minor]
    subset = all(ids < maj for ids in minor) if minor else None
    return 1.0 - voters[m] / voters.sum(), subset, dist


def device_rep(rb, W, view, obs, ring0, cfg, H, L, F, rep):
    seed, crashed, src, dst, ring, st, off = repetition(W, obs, F, rep)
    dead = np.zeros(N, np.uint8)
    dead[crashed] = 1
    cl = rb.VirtualCluster(view, H, L, kernel="sweep")
    cl.handleBatches(cfg, src, dst, ring, st, off, blocked=W.blocked_by_receiver(dead, ring0, 0, N), batch_order_seed=seed,
                     read_outputs=False)
    c = cl.proposalCensus()
    if len(c) == 0:
        cl.close()
        return []
    m = int(np.argmax(c.voters))
    d = cl.proposalCensus(cut=c.entries(m))                 # every class against the majority, on the device
    classes = [(int(d.voters[i]), frozenset(d.entries(i).tolist())) for i in range(len(d))]
    for i in range(len(d)):                                 # the device's distances are the set arithmetic summarize() does
        assert (d.missing[i], d.extra[i]) == (len(classes[m][1] - classes[i][1]), len(classes[i][1] - classes[m][1]))
    cl.close()
    return classes


def oracle_rep(orc, S, W, ow, obs, ring0, cfg, K, H, L, F, rep):
    seed, crashed, src, dst, ring, st, off = repetition(W, obs, F, rep)
    dead = np.zeros(N, np.uint8)
    dead[crashed] = 1
    sim = orc.ClusterSim(ow.view, K, H, L, N)
    _, _, props, _ = S.apply_batches(sim, src, dst, ring, st, cfg, off, blocked=dead[ring0], order_seed=seed)
    classes = {}                                            # in receiver order: first announcer = representative
    for p in props:
        if p:
            k = frozenset(p)
            classes[k] = classes.get(k, 0) + 1
    return [(v, k) for k, v in classes.items()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--oracle", action="store_true", help="run the grid on the CPU through the oracle")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from rapid_b200 import workloads as W
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
            raise SystemExit("conflict_census.py runs on the GPU (or --oracle on the CPU); no CUDA device is visible")
        import rapid_b200 as rb
        card = gpu_card()
        hb, ho, ports = W.packed_endpoints(0, N)
    table = []
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
            reps = [oracle_rep(orc, S, W, ow, obs, ring0, cfg, K, H, L, F, r) if args.oracle
                    else device_rep(rb, W, view, obs, ring0, cfg, H, L, F, r) for r in range(args.reps)]
            sums = [summarize(c) for c in reps]
            subs = [s for _, s, _ in sums if s is not None]
            dist = [d for _, _, ds in sums for d in ds]
            row = {"K": K, "H": H, "L": L, "H-L": H - L, "F": F, "reps": args.reps,
                   "disagree": float(np.mean([s[0] for s in sums])),
                   "subset": float(np.mean(subs)) if subs else None,
                   "minority_missing": float(np.mean([d[0] for d in dist])) if dist else None,
                   "minority_extra": float(np.mean([d[1] for d in dist])) if dist else None}
            fmt = lambda v: "  -  " if v is None else "%.3f" % v     # noqa: E731
            print("K=%d H=%d L=%d F=%2d  disagree %.4f  subset %s  missing %s  extra %s"
                  % (K, H, L, F, row["disagree"], fmt(row["subset"]), fmt(row["minority_missing"]), fmt(row["minority_extra"])),
                  file=sys.stderr, flush=True)
            table.append(row)
    res = {"study": "conflict_census", "nodes": N, "gpu": card, "table": table}
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
