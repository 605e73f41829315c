"""Measure the classic-Paxos fallback (SURVEY.md §8 f2) at full size: one recovery round over N virtual nodes.

    python profiles/bench_classic_paxos.py [--nodes 1000000] [--cpu-nodes 20000] [--shards W]

GPU side: rapid_b200.PaxosAcceptors / Paxos through the C ABI (wall time of each call, which includes its host
synchronisation, and the device time of the tally calls).  CPU side: the oracle's literal Paxos instances driven
message by message (one acceptor object per node, one coordinator, one learner), on a smaller N, reported per message.
--shards W also splits the N acceptors into W uneven local shards on the same GPU and reports the sharded tallies
(Paxos.handlePhase1bFromAcceptorShards / handlePhase2bFromAcceptorShards, comm-less) next to the single-handle ones, each
checked to give the single-handle result.  --cpu-nodes 0 skips the CPU side.  Prints one JSON object."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_round(n, perm_seed, n_shards=0):
    import rapid_b200 as rb
    acc = rb.PaxosAcceptors(9, n)
    ids = np.arange(n, dtype=np.int64)
    h = np.where(ids % 10 < 7, np.uint64(111), np.uint64(222)).astype(np.uint64)
    ln = np.full(n, 3, np.int32)
    out = {}
    shards = []
    if n_shards:
        # uneven pieces (sizes proportional to 1, 2, ..., W), listed last piece first
        w = np.arange(1, n_shards + 1, dtype=np.float64)
        edges = np.concatenate([[0], np.round(np.cumsum(w) / w.sum() * n)]).astype(np.int64)
        for a, b in zip(edges[:-1], edges[1:]):
            s = rb.PaxosAcceptors(9, int(b - a), acceptor_begin=int(a))
            s.registerFastRoundVotes(ids[a:b] - a, h[a:b], ln[a:b])
            shards.append(s)
        shards.reverse()
        out["shard_sizes"] = [int(s.R) for s in shards]
        sco, sle = rb.Paxos(9, n, message_capacity=n), rb.Paxos(9, n, message_capacity=n)

    def timed(name, fn):
        t0 = time.perf_counter()
        r = fn()
        out[name + "_ms"] = (time.perf_counter() - t0) * 1e3
        return r

    acc.registerFastRoundVotes(ids, h, ln)
    timed("register_votes_h2d", lambda: acc.registerFastRoundVotes(ids, h, ln))
    co, le = rb.Paxos(9, n, message_capacity=n), rb.Paxos(9, n, message_capacity=n)
    for rep in range(4):                                       # the last repetition is reported (buffers warm, handles reset)
        co.reset(9); le.reset(9)
        co.startPhase1a(2 + rep, 1)
        assert timed("acceptors_phase1a", lambda: acc.handlePhase1aMessage((2 + rep, 1))) == n
        p = timed("coordinator_phase1b", lambda: co.handlePhase1bFromAcceptors(acc, perm_seed))
        out["coordinator_phase1b_device_ms"] = co.lastDeviceMs()
        assert p.proposed and p.trigger_index == n // 2
        assert timed("acceptors_phase2a", lambda: acc.handlePhase2aMessage((2 + rep, 1), p.cval)) == n
        d = timed("learner_phase2b", lambda: le.handlePhase2bFromAcceptors(acc, perm_seed))
        out["learner_phase2b_device_ms"] = le.lastDeviceMs()
        assert d.decided and d.decided_index == n // 2 and d.decision == p.cval
        if shards:
            sco.reset(9); sle.reset(9)
            sco.startPhase1a(2 + rep, 1)
            assert sum(s.handlePhase1aMessage((2 + rep, 1)) for s in shards) == n
            sp = timed("sharded_coordinator_phase1b", lambda: sco.handlePhase1bFromAcceptorShards(shards, perm_seed=perm_seed))
            out["sharded_coordinator_phase1b_device_ms"] = sco.lastDeviceMs()
            assert (sp.proposed, sp.trigger_index, sp.cval, sp.n_messages) == (p.proposed, p.trigger_index, p.cval, p.n_messages)
            assert sum(s.handlePhase2aMessage((2 + rep, 1), p.cval) for s in shards) == n
            sd = timed("sharded_learner_phase2b", lambda: sle.handlePhase2bFromAcceptorShards(shards, perm_seed=perm_seed))
            out["sharded_learner_phase2b_device_ms"] = sle.lastDeviceMs()
            assert (sd.decided, sd.decided_index, sd.decision) == (d.decided, d.decided_index, d.decision)
    out["round_ms"] = sum(out[k] for k in ("acceptors_phase1a_ms", "coordinator_phase1b_ms", "acceptors_phase2a_ms", "learner_phase2b_ms"))
    out["messages"] = 4 * n                                    # N x (1a delivery, 1b, 2a delivery, 2b at one learner)
    out["messages_per_s"] = out["messages"] / (out["round_ms"] * 1e-3)
    return out


def cpu_round(n):
    from oracle import oracle_py as orc
    orc.build()
    u = orc.Universe()
    tags = [u.add("n", i) for i in range(n)]
    px = [orc.ClassicPaxos(u, tags[i], i + 5, 9, n) for i in range(n)]
    a, b = [tags[0], tags[1], tags[2]], [tags[3], tags[4], tags[5]]
    for i in range(n):
        px[i].registerFastRoundVote(a if i % 10 < 7 else b)
    t0 = time.perf_counter()
    m1a = px[n - 1].startPhase1a(2)
    replies = [px[i].handlePhase1aMessage(m1a) for i in range(n)]
    t1 = time.perf_counter()
    m2a = None
    for r in replies:
        o = px[n - 1].handlePhase1bMessage(r)
        if o is not None:
            m2a = o
    t2 = time.perf_counter()
    acks = [px[i].handlePhase2aMessage(m2a) for i in range(n)]
    t3 = time.perf_counter()
    for k in acks:
        px[0].handlePhase2bMessage(k)
    t4 = time.perf_counter()
    assert px[0].decided() and px[0].decision() == a
    return {"nodes": n, "acceptors_phase1a_ms": (t1 - t0) * 1e3, "coordinator_phase1b_ms": (t2 - t1) * 1e3,
            "acceptors_phase2a_ms": (t3 - t2) * 1e3, "learner_phase2b_ms": (t4 - t3) * 1e3, "round_ms": (t4 - t0) * 1e3,
            "messages": 4 * n, "messages_per_s": 4 * n / (t4 - t0),
            "note": "literal Paxos objects driven through ctypes, 1 thread; includes ~1-2 us of ctypes overhead per message"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=1_000_000)
    ap.add_argument("--cpu-nodes", type=int, default=20_000)
    ap.add_argument("--perm-seed", type=int, default=12345)
    ap.add_argument("--shards", type=int, default=0)
    args = ap.parse_args()
    res = {"nodes": args.nodes, "shards": args.shards, "gpu": gpu_round(args.nodes, args.perm_seed, args.shards),
           "gpu_acceptor_order": gpu_round(args.nodes, 0, args.shards)}
    if args.cpu_nodes > 0:
        res["cpu_oracle"] = cpu_round(args.cpu_nodes)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
