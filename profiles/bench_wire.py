"""Measure the wire-format ingest (SURVEY.md §8 f3): one serialized BatchedAlertMessage of the C5 shape (10^5 single-ring
AlertMessages over a 10^6-node view) decoded on the device, steady state, against the protobuf runtime (upb, C) parsing
the same bytes on one host core.

    python profiles/bench_wire.py [--nodes 1000000] [--messages 100000]
    python profiles/bench_wire.py --consensus [--nodes 1000000] [--messages 10000] [--vval 100] [--big 50000]
--consensus: a Phase1b inbox (--messages RapidRequests, each a --vval-endpoint vval, plus one --big-endpoint message) decoded
on the device (rapid_wire_decode_consensus) and handed to the coordinator (rapid_px_phase1b_wire), against the runtime parsing
the same bytes and fingerprinting every vval (Endpoint -> id by a dict, then rapid_proposal_fingerprint) on one host core.
Prints one JSON object."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=1_000_000)
    ap.add_argument("--messages", type=int, default=None)
    ap.add_argument("--consensus", action="store_true")
    ap.add_argument("--vval", type=int, default=100)
    ap.add_argument("--big", type=int, default=50_000)
    args = ap.parse_args()
    if args.consensus:
        return consensus(args)
    args.messages = args.messages or 100_000
    import rapid_b200 as rb
    from rapid_b200 import workloads as W
    import wire_proto
    from wire_proto import field, varint
    pb = wire_proto.build()
    n, M, K = args.nodes, args.messages, 10
    hb, off, ports = W.packed_endpoints(0, n)
    view = rb.MembershipView.from_packed(K, hb, off, ports)
    rng = np.random.default_rng(1)
    subj, obs, rings = rng.integers(0, n, M), rng.integers(0, n, M), rng.integers(0, K, M)
    hosts, ports_l = W.endpoints(0, n)
    parts = []
    for o, s, r in zip(obs.tolist(), subj.tolist(), rings.tolist()):
        alert = (field(1, 2, field(1, 2, hosts[o]) + field(2, 0, varint(int(ports_l[o])))) +
                 field(2, 2, field(1, 2, hosts[s]) + field(2, 0, varint(int(ports_l[s])))) +
                 field(3, 0, varint(1)) + field(4, 0, varint(42)) + field(5, 2, varint(r)))
        parts.append(field(3, 2, alert))
    data = b"".join(parts)
    dec = rb.WireDecoder(view)
    wall, dev = [], []
    for _ in range(6):
        t0 = time.perf_counter()
        got = dec.decodeBatchedAlertMessage(data)
        wall.append((time.perf_counter() - t0) * 1e3)
        dev.append(dec.lastDeviceMs())
    assert got.n_cells == M
    _, dst, _, _, _ = dec.cells()
    assert (dst == subj).all()
    cpu = []
    for _ in range(3):
        t0 = time.perf_counter()
        msg = pb.BatchedAlertMessage.FromString(data)
        cpu.append((time.perf_counter() - t0) * 1e3)
    # the runtime only builds objects; the reference additionally looks every Endpoint up (MembershipService.java:653-664)
    res = {"nodes": n, "messages": M, "bytes": len(data),
           "gpu_wall_ms": min(wall[1:]), "gpu_device_ms": min(dev[1:]), "gpu_first_call_ms": wall[0],
           "gpu_messages_per_s": M / (min(wall[1:]) * 1e-3), "gpu_MB_per_s": len(data) / (min(wall[1:]) * 1e-3) / 1e6,
           "cpu_protobuf_runtime_parse_ms": min(cpu), "cpu_messages_per_s": M / (min(cpu) * 1e-3),
           "cpu_note": "google.protobuf %s (upb) FromString on one core: parse only, no Endpoint -> id lookups, no cell expansion" % __import__("google.protobuf").protobuf.__version__,
           "n_messages_parsed_by_runtime": len(msg.messages)}
    print(json.dumps(res, indent=1))


def consensus(args):
    import rapid_b200 as rb
    from rapid_b200 import workloads as W
    import wire_proto_consensus as WPC
    n, M, V, K = args.nodes, args.messages or 10_000, args.vval, 10
    hb, off, ports = W.packed_endpoints(0, n)
    view = rb.MembershipView.from_packed(K, hb, off, ports)
    hosts, ports_l = W.endpoints(0, n)
    rng = np.random.default_rng(2)
    enc = {}

    def ep(j):
        if j not in enc:
            enc[j] = WPC.enc_endpoint(hosts[j], int(ports_l[j]))
        return enc[j]
    msgs = []
    for i in range(M + 1):
        size = args.big if i == M // 2 else V
        vval = np.sort(rng.choice(n, size, replace=False)).tolist()
        body = WPC.enc_message(WPC.PHASE1B, ep(int(rng.integers(0, n))), 5, (2, 1), (1, 1), WPC.enc_list(WPC.PHASE1B, [ep(j) for j in vval]))
        msgs.append(WPC.enc_request(WPC.PHASE1B, body))
    nbytes = sum(len(m) for m in msgs)
    dec = rb.WireDecoder(view)
    dev, tally, wall = [], [], []
    for _ in range(6):
        px = rb.Paxos(5, 2 * (M + 1), message_capacity=M + 1)       # N / 2 > M: every message is appended, no proposal yet
        px.startPhase1a(2, 1)
        t0 = time.perf_counter()
        dec.decodeConsensusMessages(WPC.PHASE1B, msgs, is_request=True)
        r = px.handlePhase1bFromWire(dec)
        wall.append((time.perf_counter() - t0) * 1e3)
        dev.append(dec.lastDeviceMs())
        tally.append(px.lastDeviceMs())
        assert r.n_messages == M + 1
    out = dec.consensusMessages()
    assert int(out["len"].sum()) == M * V + args.big
    pb = WPC.build()
    ids = {(h, int(p)): i for i, (h, p) in enumerate(zip(hosts, ports_l.tolist()))}
    cpu = []
    for _ in range(2):
        t0 = time.perf_counter()
        fps = []
        for m in msgs:
            x = pb.RapidRequest.FromString(m).phase1bMessage
            fps.append(rb.proposal_fingerprint([ids.get((e.hostname, e.port), -1) for e in x.vval]))
        cpu.append((time.perf_counter() - t0) * 1e3)
    assert fps[0] == (int(out["hash"][0]), int(out["hash2"][0]))
    res = {"mode": "consensus", "nodes": n, "messages": M + 1, "vval": V, "big_vval": args.big, "bytes": nbytes,
           "gpu_decode_device_ms": min(dev[1:]), "gpu_phase1b_wire_device_ms": min(tally[1:]),
           "gpu_wall_ms_decode_plus_tally": min(wall[1:]),
           "cpu_runtime_parse_and_fingerprint_ms": min(cpu),
           "cpu_note": "google.protobuf %s (upb) FromString + Endpoint -> id dict + rapid_proposal_fingerprint per message, one core"
                       % __import__("google.protobuf").protobuf.__version__}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
