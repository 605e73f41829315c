"""GPU parity of the wire-format egress (csrc/wire_encode.cu, through the C ABI) against the protobuf runtime: every message the
device encodes for a failure-detector interval or a detector's fast-round votes must equal, byte for byte, the deterministic
serialization of the message built with the runtime from the same fields, set the way MembershipService / FastPaxos set them;
and decoding what was encoded must give back what was encoded from."""
import random

import numpy as np
import pytest

import wire_proto

pytestmark = pytest.mark.gpu

K = 10


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


@pytest.fixture(scope="module")
def pb():
    return wire_proto.build()


def endpoints(n, seed):
    """n distinct endpoints whose first few stress the encoding: hostnames of 0, 1, 127, 128 and 300 bytes (varint length
    prefixes of one and two bytes), ports 0, 65535 and negative ones (10-byte varints)"""
    rng = random.Random(seed)
    special = [(b"", 0), (b"x", 65535), (b"a" * 127, -7), (b"b" * 128, 5), (b"c" * 300, 0), (b"", -2147483648)]
    hosts, ports = [], []
    for i in range(n):
        if i < len(special):
            h, p = special[i]
        else:
            h, p = b"10.%d.%d.%d" % (i >> 16, (i >> 8) & 255, i & 255), rng.choice([1, 5000 + i, -(i + 1)])
        hosts.append(h)
        ports.append(p)
    return hosts, ports


def node_ids(first, n):
    """distinct NodeIds with zero and negative halves"""
    hi = np.array([0 if i % 3 == 0 else -7 * (i + 1) for i in range(first, first + n)], np.int64)
    lo = np.array([i if i % 2 == 0 else -i for i in range(first, first + n)], np.int64)
    return hi, lo


def pb_endpoint(pb, hosts, ports, i):
    e = pb.Endpoint()
    if hosts[i]:
        e.hostname = hosts[i]
    e.port = int(ports[i])
    return e


def set_msg(field, value):
    field.SetInParent()                   # a set submessage is serialized even when it is empty
    field.MergeFrom(value)


# (H, L) of the detectors whose votes are encoded, by ring count
HL = {3: (3, 1), 10: (9, 4), 14: (12, 5)}


class Cluster:
    def __init__(self, rb, n, n_joiners, seed, K=K):
        hosts, ports = endpoints(n + n_joiners, seed)
        self.hosts, self.ports = hosts, ports
        self.K, (self.H, self.L) = K, HL[K]
        self.view = rb.MembershipView(K, hosts[:n], ports[:n])
        self.hi, self.lo = node_ids(0, n + n_joiners)
        self.view.setNodeIds(self.hi[:n], self.lo[:n])
        self.joiners = []
        if n_joiners:
            self.joiners = self.view.registerJoiners(hosts[n:], ports[n:])
            self.view.setJoinerIds(self.joiners[0], self.hi[n:], self.lo[n:])
        self.n = n

    def ep(self, pb, i):
        return pb_endpoint(pb, self.hosts, self.ports, i)


def interval(rb, c, seed, crashed_frac, tick_cfg, merge_cfg, n_leavers):
    """two failure-detector ticks (the second one fires every detector of a crashed subject), then join and leave alerts"""
    rng = random.Random(seed)
    fd = rb.EdgeFailureDetectors(c.view, failure_threshold=1)
    flags = np.zeros(c.n, np.uint8)
    crashed = rng.sample(range(c.n), max(1, int(c.n * crashed_frac)))
    flags[crashed] = rb.failure_detector.CRASHED
    fd.tick(flags, tick_cfg)
    fd.tick(flags, tick_cfg)
    live = [i for i in range(c.n) if not flags[i]]
    fd.mergeAlerts(c.joiners, rng.sample(live, n_leavers), merge_cfg)
    return fd


def expected_batches(pb, c, fd):
    """one BatchedAlertMessage per sender, alerts as MembershipService builds them (:245-253 UP, :486-492 DOWN)"""
    alerts = fd.alerts()
    _, _, _, status, cfg = fd.cells()
    out, at = [], 0
    for o, s, rings in alerts:
        if not out or out[-1][0] != o:
            b = pb.BatchedAlertMessage()
            set_msg(b.sender, c.ep(pb, o))
            out.append((o, b))
        m = out[-1][1].messages.add()
        set_msg(m.edgeSrc, c.ep(pb, o))
        set_msg(m.edgeDst, c.ep(pb, s))
        m.edgeStatus = int(status[at])
        m.configurationId = int(cfg[at])
        m.ringNumber.extend(rings)
        if status[at] == 0:
            set_msg(m.nodeId, pb.NodeId(high=int(c.hi[s]), low=int(c.lo[s])))
            m.metadata.SetInParent()
        at += len(rings)
    return out


def wrap(pb, case, msg):
    r = pb.RapidRequest()
    set_msg(getattr(r, case), msg)
    return r


def _ids(cases):
    """the ids pytest gives the cases at K = 10, with the ring count appended at the others"""
    return ["-".join(str(x) for x in c[:-1]) + ("" if c[-1] == K else "-K%d" % c[-1]) for c in cases]


# K = 3 and 14; seed 4 is a two-member view at K = 14, where the live member observes the crashed one on every ring and its
# DOWN alert lists all 14 ring numbers
ALERT_CASES = [(0, False, 0, 0, K), (1, True, -5, -5, K), (2, False, 7, -(1 << 62), K), (3, True, 1 << 40, 3, K),
               (0, False, 0, 0, 3), (1, True, -5, -5, 3), (0, False, 0, 0, 14), (1, True, -5, -5, 14), (4, False, 9, 9, 14)]


@pytest.mark.parametrize("seed,as_request,tick_cfg,merge_cfg,Kx", ALERT_CASES, ids=_ids(ALERT_CASES))
def test_alert_batches_are_byte_identical_and_decode_back(rb, pb, seed, as_request, tick_cfg, merge_cfg, Kx):
    c = Cluster(rb, [60, 400, 2000, 300, 2][seed], 4, seed, Kx)
    fd = interval(rb, c, seed, 0.05, tick_cfg, merge_cfg, n_leavers=3 if c.n > 2 else 0)
    dec = rb.WireDecoder(c.view)
    enc = dec.encodeAlertBatches(fd, as_request=as_request)
    want = expected_batches(pb, c, fd)
    assert len(enc) == len(want) > 0
    assert any(m.edgeStatus == 0 for _, b in want for m in b.messages)          # join alerts present
    if seed == 4:
        assert max(len(m.ringNumber) for _, b in want for m in b.messages) == Kx     # one alert lists every ring
    assert (enc.body_ids == -1).all() and len(enc.body_off) == 1
    for i, (_, b) in enumerate(want):
        w = wrap(pb, "batchedAlertMessage", b) if as_request else b
        assert enc.message(i) == w.SerializeToString(deterministic=True), i
    assert enc.sizes().tolist() == [len(enc.message(i)) for i in range(len(enc))]
    # round trip: the encoded batches, decoded per sender, give back the interval's cells array for array
    got = [[] for _ in range(5)]
    for i in range(len(enc)):
        dec.decodeBatchedAlertMessage(enc.message(i), is_request=as_request)
        for g, a in zip(got, dec.cells()):
            g.append(a)
    for g, a in zip(got, fd.cells()):
        assert np.array_equal(np.concatenate(g), a)


def run_votes(rb, c, seed, split):
    """one batch of an interval's cells to every receiver; split: the cells about each subject reach a random 70 % of the
    receivers, so receivers announce different subsets of the crashed nodes"""
    fd = interval(rb, c, seed, 0.04, 11, 11, n_leavers=0)
    src, dst, ring, status, cfg = fd.cells()
    vc = rb.VirtualCluster(c.view, c.H, c.L, kernel="sweep" if split else "auto")
    bitmap = None
    if split:
        rng = np.random.default_rng(seed)
        words = (vc.R + 31) // 32
        per_subject = (rng.random((c.n, words, 32)) < 0.7).astype(np.uint64)
        bits = per_subject[dst]                                                         # bit r & 31 of word r >> 5
        bitmap = (bits << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32)
    res = vc.handleBatch(11, src, dst, ring, status, bitmap=bitmap)
    return vc, res


VOTE_CASES = [(0, False, 11, False, K), (1, True, -3, False, K), (2, False, 0, True, K), (3, True, 1 << 50, True, K),
              (0, False, 11, False, 3), (2, False, 0, True, 3), (1, True, -3, False, 14), (3, True, 1 << 50, True, 14)]


@pytest.mark.parametrize("seed,as_request,cfg,split,Kx", VOTE_CASES, ids=_ids(VOTE_CASES))
def test_votes_are_byte_identical_share_bodies_and_decode_back(rb, pb, seed, as_request, cfg, split, Kx):
    c = Cluster(rb, [300, 1000, 200, 500][seed], 0, seed, Kx)
    vc, res = run_votes(rb, c, seed, split)
    voters = np.nonzero(res.proposal_len > 0)[0]
    assert len(voters) > 0
    dec = rb.WireDecoder(c.view)
    enc = dec.encodeVotes(vc, cfg, as_request=as_request)
    proposals = check_votes(pb, c, vc, voters, enc, cfg, as_request)
    if split:
        assert len(proposals) > 1
    # round trip: senders, configuration and fingerprints as the detector's outputs
    ring0 = c.view.getRing(0)
    s, cf, h1, h2, ln = dec.decodeFastRoundPhase2bMessages([enc.message(i) for i in range(len(enc))], is_request=as_request)
    assert s.tolist() == [int(ring0[r]) for r in voters]
    assert (cf == cfg).all()
    assert np.array_equal(h1, res.proposal_hash[voters]) and np.array_equal(h2, res.proposal_hash2[voters])
    assert np.array_equal(ln, res.proposal_len[voters])


def check_votes(pb, c, vc, voters, enc, cfg, as_request):
    """every vote byte-identical to the runtime's -> {proposal: its body}"""
    assert len(enc) == len(voters)
    ring0 = c.view.getRing(0)
    proposals = {}
    for i, r in enumerate(voters):
        ids = vc.getProposal(int(r))
        v = pb.FastRoundPhase2bMessage()
        set_msg(v.sender, c.ep(pb, int(ring0[r])))
        v.configurationId = cfg
        for j in ids:
            v.endpoints.add().MergeFrom(c.ep(pb, j))
        w = wrap(pb, "fastRoundPhase2bMessage", v) if as_request else v
        assert enc.message(i) == w.SerializeToString(deterministic=True), (i, r)
        proposals.setdefault(tuple(ids), int(enc.body_ids[i]))
    # one body per distinct proposal, numbered by its lowest receiver, each the encoding of that proposal's list
    assert len(enc.body_off) - 1 == len(proposals) == len(set(proposals.values()))
    assert sorted(proposals.values()) == list(range(len(proposals)))
    for ids, b in proposals.items():
        assert enc.body(b) == b"".join(wire_proto.field(3, 2, c.ep(pb, j).SerializeToString(deterministic=True)) for j in ids)
    assert enc.sizes().sum() == sum(len(enc.message(i)) for i in range(len(enc)))
    return proposals


def census_state(vc, census, cut_len):
    """what a user reads of the detector's last census"""
    from rapid_b200.cut_detector import ProposalCensus
    c = ProposalCensus(vc, len(census), len(census.ids), cut_len)
    return ([a.tobytes() for a in (c.hash, c.hash2, c.length, c.voters, c.representative, c.in_cut, c.list_off, c.ids, c.status,
                                   c.classes())], c.classes_dev)


@pytest.mark.parametrize("as_request", [False, True])
def test_encoding_votes_leaves_the_detectors_census(rb, pb, as_request):
    """the vote encode lists the proposals in storage of its own: the census taken before it reads back unchanged after it"""
    c = Cluster(rb, 1000, 0, 1)
    vc, res = run_votes(rb, c, 1, True)
    voters = np.nonzero(res.proposal_len > 0)[0]
    cut = np.unique(np.concatenate([vc.getProposal(int(r)) for r in voters[:3]]))
    census = vc.proposalCensus(cut)
    assert len(census) > 1 and (census.in_cut >= 0).all()
    before = census_state(vc, census, len(cut))
    enc = rb.WireDecoder(c.view).encodeVotes(vc, 5, as_request=as_request)
    assert census_state(vc, census, len(cut)) == before
    proposals = check_votes(pb, c, vc, voters, enc, 5, as_request)
    assert len(proposals) == len(census)


def snapshot(dec):
    e = dec.encoded()
    return (e.headers.tobytes(), e.header_off.tobytes(), e.body_ids.tobytes(), e.bodies.tobytes(), e.body_off.tobytes(),
            e.sizes().tobytes())


def test_refusals_leave_the_last_encode_and_the_decode(rb, pb):
    c = Cluster(rb, 200, 0, 7)
    vc, _ = run_votes(rb, c, 7, False)
    dec = rb.WireDecoder(c.view)
    enc = dec.encodeVotes(vc, 11)
    dec.decodeFastRoundPhase2bMessages([enc.message(i) for i in range(len(enc))])
    cons = dec.consensusMessages()
    before = snapshot(dec)
    other = Cluster(rb, 200, 0, 8)
    fresh_fd = rb.EdgeFailureDetectors(c.view)                                    # no interval since its reset
    ticked_other = interval(rb, other, 8, 0.05, 0, 0, 0)                          # another view
    refusals = [lambda: dec.encodeVotes(rb.VirtualCluster(c.view, 9, 4), 11),     # a detector that applied no batch
                lambda: dec.encodeVotes(run_votes(rb, other, 8, False)[0], 11),  # another view
                lambda: dec.encodeAlertBatches(fresh_fd),
                lambda: dec.encodeAlertBatches(ticked_other)]
    for f in refusals:
        with pytest.raises(rb.RapidError):
            f()
        assert snapshot(dec) == before
        after = dec.consensusMessages()
        assert all(np.array_equal(after[k], cons[k]) for k in cons)


def test_a_decode_between_encodes_leaves_the_encode(rb, pb):
    c = Cluster(rb, 300, 2, 9)
    fd = interval(rb, c, 9, 0.05, 4, 4, 1)
    dec = rb.WireDecoder(c.view)
    enc = dec.encodeAlertBatches(fd, as_request=True)
    before = snapshot(dec)
    dec.decodeBatchedAlertMessage(enc.message(0), is_request=True)
    assert snapshot(dec) == before


def test_scale_sizes_sum_to_the_bytes_written(rb, pb):
    n = 20000
    c = Cluster(rb, n, 0, 11)
    fd = interval(rb, c, 11, 0.01, 42, 42, 0)
    dec = rb.WireDecoder(c.view)
    enc = dec.encodeAlertBatches(fd, as_request=True)
    counts = dec.encodedCounts()
    assert enc.sizes().sum() == counts[1] + counts[3] == len(enc.headers)
    rng = random.Random(0)
    for i in rng.sample(range(len(enc)), 50):
        r = pb.RapidRequest()
        r.ParseFromString(enc.message(i))
        assert r.SerializeToString(deterministic=True) == enc.message(i)
    vc = rb.VirtualCluster(c.view, 9, 4)
    src, dst, ring, status, cfg = fd.cells()
    res = vc.handleBatch(42, src, dst, ring, status)
    enc = dec.encodeVotes(vc, 42, as_request=True)
    counts = dec.encodedCounts()
    assert len(enc) == int((res.proposal_len > 0).sum()) > n // 2
    assert counts[2] == 1 and enc.sizes().sum() == counts[1] + len(enc) * counts[3]
    for i in rng.sample(range(len(enc)), 50):
        r = pb.RapidRequest()
        r.ParseFromString(enc.message(i))
        assert len(r.fastRoundPhase2bMessage.endpoints) == res.proposal_len.max()


@pytest.fixture(scope="module")
def pc():
    import wire_proto_consensus
    return wire_proto_consensus.build()


def set_rank(field, rk):
    field.SetInParent()                   # Paxos sets rnd / vrnd always: written even when (0, 0)
    field.round, field.nodeIndex = int(rk[0]), int(rk[1])


@pytest.mark.parametrize("seed,as_request,via_cache", [(0, False, True), (1, True, False)])
def test_phase1b_and_phase2b_answers_are_byte_identical_and_tally_as_from_the_acceptors(rb, pb, pc, seed, as_request, via_cache):
    """the acceptors' answers of a classic round over a split fast round: byte identity with the runtime, decode round trip, and
    the *_wire tallies over the decoded answers decide exactly as the tallies over the acceptors"""
    c = Cluster(rb, [200, 500][seed], 0, seed)
    vc, res = run_votes(rb, c, seed, True)
    n, cfg, rank = c.n, -9 if seed else 11, (2, -5)
    acc = rb.PaxosAcceptors(cfg, n)
    acc.registerFastRoundVotesFrom(vc)
    silent = np.zeros(n, np.uint8)
    silent[random.Random(seed).sample(range(n), n // 10)] = 1
    acc.setSilent(silent)
    dec = rb.WireDecoder(c.view)
    if via_cache:
        dec.encodeVotes(vc, cfg)                                              # the votes carried every list the acceptors hold
    acc.handlePhase1aMessage(rank, msg_cfg=cfg)
    enc = dec.encodePhase1b(acc, None if via_cache else vc, as_request=as_request)
    ring0 = c.view.getRing(0)
    answering = [r for r in range(n) if not silent[r]]
    assert len(enc) == len(answering)
    states = [acc.read(r) for r in answering]
    assert any(s["vval"][2] == 0 for s in states) and any(s["vval"][2] > 0 for s in states)   # empty and non-empty vvals
    for i, (r, st) in enumerate(zip(answering, states)):
        m = pc.Phase1bMessage()
        set_msg(m.sender, pc.Endpoint(hostname=c.hosts[int(ring0[r])], port=int(c.ports[int(ring0[r])])))
        m.configurationId = cfg
        set_rank(m.rnd, rank)
        set_rank(m.vrnd, st["vrnd"])
        for j in (vc.getProposal(r) if st["vval"][2] else []):
            m.vval.add().MergeFrom(pc.Endpoint(hostname=c.hosts[j], port=int(c.ports[j])))
        w = pc.RapidRequest(phase1bMessage=m) if as_request else m
        assert enc.message(i) == w.SerializeToString(deterministic=True), (i, r)
        assert enc.senders[i] == ring0[r]
    assert enc.sizes().sum() == sum(len(enc.message(i)) for i in range(len(enc)))
    # round trip and tally
    px_dev, px_wire = rb.Paxos(cfg, n), rb.Paxos(cfg, n)
    for px in (px_dev, px_wire):
        px.startPhase1a(*rank)
    want1 = px_dev.handlePhase1bFromAcceptors(acc)
    dec.decodeConsensusMessages(rb._native.WIRE_PHASE1B, [enc.message(i) for i in range(len(enc))], is_request=as_request)
    got = dec.consensusMessages()
    assert got["sender"].tolist() == [int(ring0[r]) for r in answering]
    assert [(int(a), int(b), int(l)) for a, b, l in zip(got["hash"], got["hash2"], got["len"])] == [s["vval"] for s in states]
    have1 = px_wire.handlePhase1bFromWire(dec)
    assert (have1.proposed, have1.trigger_index, have1.cval) == (want1.proposed, want1.trigger_index, want1.cval)
    assert want1.proposed
    proposer = acc.findValue(want1.cval)
    acc.handlePhase2aMessage(rank, want1.cval, msg_cfg=cfg)
    enc2 = dec.encodePhase2b(acc, None if via_cache else vc, as_request=as_request)
    value = vc.getProposal(proposer)
    assert len(enc2) == len(answering) and (enc2.body_ids == 0).all() and len(enc2.body_off) == 2
    for i, r in enumerate(answering):
        m = pc.Phase2bMessage()
        set_msg(m.sender, pc.Endpoint(hostname=c.hosts[int(ring0[r])], port=int(c.ports[int(ring0[r])])))
        m.configurationId = cfg
        set_rank(m.rnd, rank)
        for j in value:
            m.endpoints.add().MergeFrom(pc.Endpoint(hostname=c.hosts[j], port=int(c.ports[j])))
        w = pc.RapidRequest(phase2bMessage=m) if as_request else m
        assert enc2.message(i) == w.SerializeToString(deterministic=True), (i, r)
    want2 = px_dev.handlePhase2bFromAcceptors(acc)
    dec.decodeConsensusMessages(rb._native.WIRE_PHASE2B, [enc2.message(i) for i in range(len(enc2))], is_request=as_request)
    have2 = px_wire.handlePhase2bFromWire(dec)
    assert (have2.decided, have2.decided_index, have2.decision) == (want2.decided, want2.decided_index, want2.decision)
    assert want2.decided


def test_encoded_votes_tally_as_the_detector_outputs(rb, pb):
    """rapid_fp_tally_wire over the decoded encoded votes decides exactly as rapid_fp_tally_cd over the detector"""
    c = Cluster(rb, 400, 0, 5)
    vc, res = run_votes(rb, c, 5, False)
    dec = rb.WireDecoder(c.view)
    enc = dec.encodeVotes(vc, 11, as_request=True)
    fa, fb = rb.FastPaxos(11, c.n), rb.FastPaxos(11, c.n)
    want = fa.tallyCluster(vc)
    dec.decodeConsensusMessages(rb._native.WIRE_FAST_ROUND_PHASE2B, [enc.message(i) for i in range(len(enc))], is_request=True)
    have = fb.handleFastRoundProposalsFromWire(dec)
    assert want.decided
    for k in ("decided", "hash", "hash2", "length", "count", "votes_received"):
        assert getattr(have, k) == getattr(want, k), k


def test_refusal_of_a_detector_from_before_a_view_change(rb, pb):
    c = Cluster(rb, 300, 0, 12)
    vc, res = run_votes(rb, c, 12, False)
    dec = rb.WireDecoder(c.view)
    dec.encodeVotes(vc, 11)
    before = snapshot(dec)
    c.view.applyCut([c.n - 1])                                                # one member leaves: the ids renumber
    with pytest.raises(rb.RapidError):
        dec.encodeVotes(vc, 11)
    assert snapshot(dec) == before


def test_million_node_interval_and_votes(rb, pb):
    """the C5-shaped interval (10^6 nodes, 1 % crashed) and the 10^6 votes for its cut: a seeded sample of messages parses with
    the runtime into what the device holds, the one body is the cut of every sampled announcer, sizes sum to the bytes"""
    from rapid_b200 import workloads as W
    n = 1_000_000
    hb, off, ports = W.packed_endpoints(0, n)
    view = rb.MembershipView.from_packed(K, hb, off, ports)
    view.setNodeIds(*W.node_ids(0, n))
    fd = rb.EdgeFailureDetectors(view, failure_threshold=1)
    flags = np.zeros(n, np.uint8)
    flags[np.random.default_rng(3).choice(n, n // 100, replace=False)] = rb.failure_detector.CRASHED
    fd.tick(flags, 7)
    fd.tick(flags, 7)
    dec = rb.WireDecoder(view)
    enc = dec.encodeAlertBatches(fd, as_request=True)
    counts = dec.encodedCounts()
    assert len(enc) > 50_000 and enc.sizes().sum() == counts[1] == len(enc.headers)
    rng = random.Random(1)
    for i in rng.sample(range(len(enc)), 200):
        r = pb.RapidRequest()
        r.ParseFromString(enc.message(i))
        assert r.SerializeToString(deterministic=True) == enc.message(i)
        assert all(m.edgeStatus == 1 and m.configurationId == 7 for m in r.batchedAlertMessage.messages)
    vc = rb.VirtualCluster(view, 9, 4)
    src, dst, ring, status, cfg = fd.cells()
    res = vc.handleBatch(7, src, dst, ring, status)
    enc = dec.encodeVotes(vc, 7, as_request=True)
    voters = np.nonzero(res.proposal_len > 0)[0]
    assert len(enc) == len(voters) > n // 2 and len(enc.body_off) == 2
    assert enc.sizes().sum() == len(enc.headers) + len(enc) * len(enc.bodies)
    body = enc.body(0)
    for i in rng.sample(range(len(enc)), 100):
        r = int(voters[i])
        ids = vc.getProposal(r)
        assert body == b"".join(wire_proto.field(3, 2, pb_endpoint_packed(pb, hb, off, ports, j)) for j in ids)
        m = pb.RapidRequest()
        m.ParseFromString(enc.message(i))
        assert len(m.fastRoundPhase2bMessage.endpoints) == len(ids) == n // 100


def pb_endpoint_packed(pb, hb, off, ports, j):
    e = pb.Endpoint(hostname=bytes(hb[off[j]:off[j + 1]]), port=int(ports[j]))
    return e.SerializeToString(deterministic=True)


@pytest.mark.parametrize("frac,seed", [(0.01, 24), (0.30, 23)])
def test_cluster_simulation_wire_traffic_adds_only_wire_bytes(rb, frac, seed):
    """with wire_traffic=True every record is the default run's plus the wire keys; the 30 % draw takes the classic round, so
    its deciding interval also counts Phase1b / Phase2b answers"""
    from rapid_b200 import workloads as W
    from test_gpu_cluster_simulation import _no_dark_draw
    n = 1000
    v = rb.MembershipView.from_packed(K, *W.packed_endpoints(0, n))
    obs, _ = v.tables()
    v.close()
    crashed = _no_dark_draw(obs, n, frac, seed)
    runs = []
    for wt in (False, True):
        s = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=seed, wire_traffic=wt)
        for t in crashed:
            s.setFlags(t, rb.failure_detector.CRASHED)
        s.run(30)
        runs.append(s)
    timing = {"device_ms", "host_ms", "detect_ms", "classic_ms", "view_change_ms", "handles_ms"}
    wire = {"wire_bytes", "wire_tx_max", "wire_tx_mean", "wire_rx_max", "wire_rx_mean"}
    a, b = runs
    assert len(a.intervals) == len(b.intervals) and len(a.history) == len(b.history) >= 1
    for ra, rb_ in zip(a.intervals, b.intervals):
        assert not (set(ra) & wire) and set(rb_) - set(ra) == wire
        assert {k: v for k, v in ra.items() if k not in timing} == {k: v for k, v in rb_.items() if k not in timing | wire}
        assert (rb_["wire_bytes"] > 0) == (rb_["alerts"] > 0 or rb_["event"] == "decided-classic")
        assert rb_["wire_tx_max"] >= rb_["wire_tx_mean"] and rb_["wire_rx_max"] * 0 + rb_["wire_rx_mean"] == rb_["wire_rx_max"]
    for ha, hb_ in zip(a.history, b.history):
        assert {k: v for k, v in ha.items() if k not in timing} == {k: v for k, v in hb_.items() if k not in timing}
    if frac > 0.1:
        assert any(h["path"] == "classic" for h in b.history)
