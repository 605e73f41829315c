"""GPU parity of the consensus-message decoder (csrc/wire.cu, rapid_wire_decode_consensus) and of the tallies fed from it
without a host round trip (rapid_px_phase1b_wire / rapid_px_phase2b_wire / rapid_fp_tally_wire).  The protobuf runtime is the
encoder and the reference parser; the oracle's ClassicPaxos / FastPaxosTally and tests/plainref.py are the references for the
tallies."""
import random

import numpy as np
import pytest

import plainref
import wire_proto_consensus as WPC
from wire_proto import field, varint
from rapid_b200 import workloads as W

pytestmark = pytest.mark.gpu

K = 10
KINDS = [WPC.FAST_ROUND_PHASE2B, WPC.PHASE1A, WPC.PHASE1B, WPC.PHASE2A, WPC.PHASE2B]
INT_MIN, INT_MAX = -2**31, 2**31 - 1


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


@pytest.fixture(scope="module")
def pb():
    return WPC.build()


def make_view(rb, n, joiners=0):
    hb, off, ports = W.packed_endpoints(0, n)
    v = rb.MembershipView.from_packed(K, hb, off, ports)
    if joiners:
        v.registerJoiners(*W.endpoints(n, joiners))
    return v


def ep_of(i):
    hosts, ports = W.endpoints(i, 1)
    return bytes(hosts[0]) if not isinstance(hosts[0], str) else hosts[0].encode(), int(ports[0])


class Dict:
    """(hostname, port) -> id of the view's endpoints + registered joiners"""

    def __init__(self, total):
        hosts, ports = W.endpoints(0, total)
        self.ids = {(h if isinstance(h, bytes) else h.encode(), int(p)): i for i, (h, p) in enumerate(zip(hosts, ports.tolist()))}

    def __call__(self, e):
        return self.ids.get((bytes(e.hostname), int(e.port)), -1)


def random_message(pb, rng, kind, universe, stranger_rate=0.1):
    m = pb.kind[kind]()
    ids = []
    if rng.random() < 0.9:
        if rng.random() < stranger_rate:
            m.sender.hostname, m.sender.port = b"stranger", rng.randrange(4)
        else:
            m.sender.hostname, m.sender.port = ep_of(rng.randrange(universe))
    m.configurationId = rng.choice([0, 3, -3, 2**62, INT_MIN * 2**32, rng.getrandbits(63)])
    rk = lambda: (rng.choice([0, 1, 2, -1, INT_MIN, INT_MAX, rng.randint(INT_MIN, INT_MAX)]), rng.choice([0, 9, -9, INT_MIN, INT_MAX]))
    if WPC.RANK_NAME[kind] and rng.random() < 0.85:
        r = getattr(m, WPC.RANK_NAME[kind]); r.round, r.nodeIndex = rk()
    if kind == WPC.PHASE1B and rng.random() < 0.85:
        m.vrnd.round, m.vrnd.nodeIndex = rk()
    if WPC.LIST_NAME[kind] and rng.random() < 0.9:
        lst = getattr(m, WPC.LIST_NAME[kind])
        for _ in range(rng.choice([0, 1, 3, 12, 40])):
            if rng.random() < stranger_rate:
                lst.add(hostname=b"nobody-%d" % rng.randrange(5), port=rng.randrange(3))
            else:
                j = rng.randrange(universe)
                if ids and rng.random() < 0.1:
                    j = ids[0]                                             # a duplicate endpoint
                lst.add(hostname=ep_of(j)[0], port=ep_of(j)[1])
                ids.append(j)
    return m


def expected(pb, m, kind, id_of):
    rank = getattr(m, WPC.RANK_NAME[kind]) if WPC.RANK_NAME[kind] else None
    vr = m.vrnd if kind == WPC.PHASE1B else None
    lst = list(getattr(m, WPC.LIST_NAME[kind])) if WPC.LIST_NAME[kind] else []
    return {"sender": id_of(m.sender) if m.HasField("sender") else -1, "cfg": m.configurationId,
            "rnd_round": rank.round if rank is not None else 0, "rnd_node": rank.nodeIndex if rank is not None else 0,
            "vrnd_round": vr.round if vr is not None else 0, "vrnd_node": vr.nodeIndex if vr is not None else 0,
            "ids": [id_of(e) for e in lst], "list": lst}


def fingerprint_of_list(rb, dec, pb, ids, lst):
    """what the decoder must give a list: rapid_proposal_fingerprint when every endpoint is known, else the fingerprint
    the vote decoder gives the same list"""
    if all(i >= 0 for i in ids):
        return rb.proposal_fingerprint(ids)
    v = pb.FastRoundPhase2bMessage()
    v.endpoints.extend(lst)
    _, _, h1, h2, _ = dec.decodeFastRoundPhase2bMessages([v.SerializeToString()])
    return int(h1[0]), int(h2[0])


def serialize(pb, kind, m, as_request):
    return pb.RapidRequest(**{WPC.CASES[kind]: m}).SerializeToString() if as_request else m.SerializeToString()


# ------------------------------------------------------------------------------------------------ 1. field by field
@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("as_request", [False, True])
def test_fields_match_the_runtime_for_every_kind(rb, pb, seed, as_request):
    n = 300
    view = make_view(rb, n, joiners=5)
    id_of = Dict(n + 5)
    dec, ref = rb.WireDecoder(view), rb.WireDecoder(view)
    rng = random.Random(seed * 10 + as_request)
    for kind in KINDS:
        msgs = [random_message(pb, rng, kind, n + 5) for _ in range(rng.choice([1, 50, 200]))]
        data = [serialize(pb, kind, m, as_request) for m in msgs]
        for d, m in zip(data, msgs):                                    # the runtime parses back what it wrote
            got = pb.RapidRequest.FromString(d) if as_request else pb.kind[kind].FromString(d)
            assert (getattr(got, WPC.CASES[kind]) if as_request else got) == m
        us, ue = dec.decodeConsensusMessages(kind, data, is_request=as_request)
        out = dec.consensusMessages()
        want = [expected(pb, m, kind, id_of) for m in msgs]
        assert us == sum(1 for w in want if w["sender"] < 0)
        assert ue == sum(1 for w in want for i in w["ids"] if i < 0)
        for key in ("sender", "cfg", "rnd_round", "rnd_node", "vrnd_round", "vrnd_node"):
            assert out[key].tolist() == [w[key] for w in want], (kind, key)
        assert out["len"].tolist() == [len(w["ids"]) for w in want]
        for i, w in enumerate(want):
            assert dec.consensusValue(i) == w["ids"]
            h = fingerprint_of_list(rb, ref, pb, w["ids"], w["list"])
            assert (int(out["hash"][i]), int(out["hash2"][i])) == h, (kind, i)


# ------------------------------------------------------------------------------------------------ 2. hand-rolled encodings
def test_encodings_the_runtime_never_emits(rb, pb):
    n = 40
    view = make_view(rb, n)
    dec = rb.WireDecoder(view)
    e = lambda i: WPC.enc_endpoint(*ep_of(i))
    cases = []
    # Rank twice: merged field by field (round from the first, nodeIndex from the second)
    b = field(3, 2, field(1, 0, varint(7))) + field(3, 2, field(2, 0, varint(-4))) + field(1, 2, e(3))
    cases.append((WPC.PHASE1A, b))
    # a rank varint with bits above 32: the low 32 bits
    cases.append((WPC.PHASE2A, field(3, 2, field(1, 0, varint((5 << 32) | 9)) + field(2, 0, varint(-1))) + field(5, 2, e(1))))
    # a wire-type mismatch on round: skipped as an unknown field; nodeIndex still read
    cases.append((WPC.PHASE1B, field(3, 2, field(1, 2, b"xx") + field(2, 0, varint(6))) + field(4, 2, field(1, 0, varint(2)))))
    # unknown fields of every wire type (top level and inside Rank / Endpoint), fields out of order, a second sender merged
    b = (field(5, 2, e(2)) + field(99, 0, varint(1 << 40)) + field(98, 1, b"12345678") + field(97, 5, b"1234") + field(96, 2, b"junk") +
         field(3, 2, field(9, 5, b"abcd") + field(1, 0, varint(3))) + field(2, 0, varint(-9)) + field(1, 2, field(2, 0, varint(ep_of(4)[1]))) +
         field(5, 2, e(0) + field(50, 0, varint(1))) + field(1, 2, field(1, 2, ep_of(4)[0])) + field(4, 2, b""))
    cases.append((WPC.PHASE1B, b))
    # a Phase2b list sent as field 5 is skipped (len 0); a Phase1b list as field 4 is a Rank (vrnd) — here an empty one
    cases.append((WPC.PHASE2B, field(5, 2, e(1)) + field(5, 2, e(2)) + field(2, 0, varint(4))))
    cases.append((WPC.PHASE1B, field(4, 2, b"") + field(5, 2, e(6))))
    cases.append((WPC.FAST_ROUND_PHASE2B, field(3, 0, varint(4)) + field(3, 2, e(8))))      # wire-type mismatch on a list
    for kind, raw in cases:
        want = pb.kind[kind].FromString(raw)                            # the runtime accepts these
        id_of = Dict(n)
        dec.decodeConsensusMessages(kind, [raw])
        out = dec.consensusMessages()
        w = expected(pb, want, kind, id_of)
        for key in ("sender", "cfg", "rnd_round", "rnd_node", "vrnd_round", "vrnd_node"):
            assert out[key][0] == w[key], (kind, key, raw)
        assert dec.consensusValue(0) == w["ids"]
        assert (int(out["hash"][0]), int(out["hash2"][0])) == rb.proposal_fingerprint(w["ids"])
        # as a RapidRequest: twice the case merges (lists concatenate), another case later replaces it
        req = WPC.enc_request(kind, raw)
        dec.decodeConsensusMessages(kind, [req + req], is_request=True)
        merged = getattr(pb.RapidRequest.FromString(req + req), WPC.CASES[kind])
        assert dec.consensusValue(0) == expected(pb, merged, kind, id_of)["ids"]
        other = WPC.PHASE2A if kind != WPC.PHASE2A else WPC.PHASE2B
        assert pb.RapidRequest.FromString(req + WPC.enc_request(other, b"")).WhichOneof("content") == WPC.CASES[other]
        with pytest.raises(rb.RapidError, match="malformed " + WPC.NAMES[kind]):
            dec.decodeConsensusMessages(kind, [req + WPC.enc_request(other, b"")], is_request=True)
        dec.decodeConsensusMessages(kind, [WPC.enc_request(other, b"") + req], is_request=True)      # ... and back
        with pytest.raises(rb.RapidError):
            dec.decodeConsensusMessages(kind, [pb.RapidRequest(probeMessage=pb.ProbeMessage()).SerializeToString()], is_request=True)


# ------------------------------------------------------------------------------------------------ 3. refused bytes
@pytest.mark.parametrize("kind", KINDS)
def test_every_truncation_is_refused_like_the_runtime(rb, pb, kind):
    n = 30
    view = make_view(rb, n)
    dec = rb.WireDecoder(view)
    rng = random.Random(kind)
    px, fp = rb.Paxos(3, n), rb.FastPaxos(3, n)
    for _ in range(3):
        m = pb.kind[kind]()
        m.sender.hostname, m.sender.port = ep_of(1)
        m.configurationId = rng.choice([5, -5, 2**40])
        if WPC.RANK_NAME[kind]:
            r = getattr(m, WPC.RANK_NAME[kind]); r.round, r.nodeIndex = rng.choice([(2, 3), (-1, INT_MAX)])
        if kind == WPC.PHASE1B:
            m.vrnd.round, m.vrnd.nodeIndex = 1, 1
        if WPC.LIST_NAME[kind]:
            for j in rng.sample(range(n), 2):
                getattr(m, WPC.LIST_NAME[kind]).add(hostname=ep_of(j)[0], port=ep_of(j)[1])
        for as_request in (False, True):
            data = serialize(pb, kind, m, as_request)
            for cut in range(1, len(data)):
                bad = data[:cut]
                try:
                    (pb.RapidRequest if as_request else pb.kind[kind]).FromString(bad)
                    runtime_ok = True
                except Exception:
                    runtime_ok = False
                if as_request and runtime_ok and pb.RapidRequest.FromString(bad).WhichOneof("content") != WPC.CASES[kind]:
                    runtime_ok = False                                   # a request that does not carry the message
                if runtime_ok:
                    dec.decodeConsensusMessages(kind, [data, bad], is_request=as_request)
                    continue
                with pytest.raises(rb.RapidError, match="malformed %s at index 1" % WPC.NAMES[kind]):
                    dec.decodeConsensusMessages(kind, [data, bad], is_request=as_request)
                with pytest.raises(rb.RapidError):
                    dec.consensusMessages()
            # after a refused decode the tallies refuse too
            with pytest.raises(rb.RapidError):
                dec.decodeConsensusMessages(kind, [data, b"\x00"], is_request=as_request)
            with pytest.raises(rb.RapidError):
                px.handlePhase1bFromWire(dec)
            with pytest.raises(rb.RapidError):
                px.handlePhase2bFromWire(dec)
            with pytest.raises(rb.RapidError):
                fp.handleFastRoundProposalsFromWire(dec)


# ------------------------------------------------------------------------------------------------ 4. the vote decoder is kind 5
@pytest.mark.parametrize("as_request", [False, True])
def test_decode_votes_is_kind_5(rb, pb, as_request):
    n = 500
    view = make_view(rb, n, joiners=3)
    dec = rb.WireDecoder(view)
    rng = random.Random(9)
    msgs = [serialize(pb, 5, random_message(pb, rng, 5, n + 10), as_request) for _ in range(400)]
    votes = dec.decodeFastRoundPhase2bMessages(msgs, is_request=as_request)
    dec.decodeConsensusMessages(5, msgs, is_request=as_request)
    out = dec.consensusMessages()
    for a, k in zip(votes, ("sender", "cfg", "hash", "hash2", "len")):
        np.testing.assert_array_equal(a, out[k])
    assert not out["rnd_round"].any() and not out["vrnd_node"].any()


# ------------------------------------------------------------------------------------------------ 5. bit-identical to host arrays
def _p1_tuple(r):
    return (r.proposed, r.trigger_index, r.cval, r.n_messages)


def test_wire_tallies_equal_the_host_array_tallies(rb, pb):
    n, cfg = 64, 11
    view = make_view(rb, n)
    dec, id_of = rb.WireDecoder(view), Dict(n)
    rng = random.Random(5)
    values = [sorted(rng.sample(range(n), rng.randint(1, 6))) for _ in range(4)]
    # Phase1b: several calls, the list growing past message_capacity; few keep (rnd == crnd)
    a, b = rb.Paxos(cfg, n, message_capacity=8), rb.Paxos(cfg, n, message_capacity=8)
    for p in (a, b):
        p.startPhase1a(2, 5)
    for call in range(6):
        msgs = []
        for _ in range(rng.randint(0, 25)):
            m = pb.Phase1bMessage()
            m.sender.hostname, m.sender.port = ep_of(rng.randrange(n))
            m.configurationId = rng.choice([cfg, cfg, cfg, cfg + 1])
            m.rnd.round, m.rnd.nodeIndex = rng.choice([(2, 5), (2, 5), (1, 5), (2, 4)])
            m.vrnd.round, m.vrnd.nodeIndex = rng.choice([(0, 0), (1, 1), (2, 3)])
            if rng.random() < 0.8:
                for j in rng.choice(values):
                    m.vval.add(hostname=ep_of(j)[0], port=ep_of(j)[1])
            msgs.append(m)
        dec.decodeConsensusMessages(WPC.PHASE1B, [m.SerializeToString() for m in msgs])
        out = dec.consensusMessages()
        ra = a.handlePhase1bFromWire(dec)
        rb_ = b.handlePhase1bMessages(np.stack([out["rnd_round"], out["rnd_node"]], 1), np.stack([out["vrnd_round"], out["vrnd_node"]], 1),
                                      out["hash"], out["len"], vval_hash2=out["hash2"], msg_cfg=out["cfg"])
        assert _p1_tuple(ra) == _p1_tuple(rb_)
    assert a.handlePhase1bFromWire(dec).n_messages > 8
    # Phase2b, several rounds and duplicate senders
    a, b = rb.Paxos(cfg, n, message_capacity=256), rb.Paxos(cfg, n, message_capacity=256)
    for call in range(5):
        msgs = []
        for _ in range(rng.randint(0, 30)):
            m = pb.Phase2bMessage()
            m.sender.hostname, m.sender.port = ep_of(rng.randrange(n))
            m.configurationId = rng.choice([cfg, cfg, cfg + 1])
            m.rnd.round, m.rnd.nodeIndex = rng.choice([(2, 5), (3, 1)])
            for j in rng.choice(values):
                m.endpoints.add(hostname=ep_of(j)[0], port=ep_of(j)[1])
            msgs.append(m)
        dec.decodeConsensusMessages(WPC.PHASE2B, [m.SerializeToString() for m in msgs])
        out = dec.consensusMessages()
        ra = a.handlePhase2bFromWire(dec)
        rb_ = b.handlePhase2bMessages(np.stack([out["rnd_round"], out["rnd_node"]], 1), out["sender"], out["hash"], out["len"],
                                      value_hash2=out["hash2"], msg_cfg=out["cfg"])
        assert (ra.decided, ra.decided_index, ra.decision) == (rb_.decided, rb_.decided_index, rb_.decision)
    # the fast round
    fa, fb = rb.FastPaxos(cfg, n), rb.FastPaxos(cfg, n)
    for call in range(8):
        msgs = []
        for _ in range(rng.randint(0, 60)):
            m = pb.FastRoundPhase2bMessage()
            m.sender.hostname, m.sender.port = ep_of(rng.randrange(n))
            m.configurationId = rng.choice([cfg, cfg, cfg + 1])
            for j in values[0] if rng.random() < 0.9 else rng.choice(values):
                m.endpoints.add(hostname=ep_of(j)[0], port=ep_of(j)[1])
            msgs.append(m)
        dec.decodeConsensusMessages(WPC.FAST_ROUND_PHASE2B, [m.SerializeToString() for m in msgs])
        out = dec.consensusMessages()
        ra = fa.handleFastRoundProposalsFromWire(dec)
        rb_ = fb.handleFastRoundProposals(out["sender"], out["hash"], out["hash2"], out["len"], vote_cfg=out["cfg"])
        assert (ra.decided, ra.hash, ra.hash2, ra.length, ra.count, ra.votes_received) == \
            (rb_.decided, rb_.hash, rb_.hash2, rb_.length, rb_.count, rb_.votes_received)
    assert ra.decided


# ------------------------------------------------------------------------------------------------ 6. whole rounds vs the oracle
class WireNet:
    """N oracle ClassicPaxos / FastPaxosTally nodes (the PaxosTests wiring); node 0's inbox is ALSO serialized by the runtime
    and run through decode -> *_wire / rapid_pxa_* on the device, batch by batch, and compared at every batch."""

    def __init__(self, orc, rb, pb, N, seed):
        self.rb, self.pb, self.N, self.rng = rb, pb, N, random.Random(seed)
        self.cfg = 1000 + seed
        self.u = orc.Universe()
        self.tags = [self.u.add(*ep_of(i)) for i in range(N)]
        self.id_of_tag = {t: i for i, t in enumerate(self.tags)}
        hashes = list(range(100, 100 + N))
        random.Random(seed + 1).shuffle(hashes)
        self.hashes = hashes
        self.px = [orc.ClassicPaxos(self.u, self.tags[i], hashes[i], self.cfg, N) for i in range(N)]
        self.fp = [orc.FastPaxosTally(self.u, self.cfg, N) for _ in range(N)]
        self.inbox = [[] for _ in range(N)]
        self.view = make_view(rb, N)
        self.dec = rb.WireDecoder(self.view)
        self.dpx = rb.Paxos(self.cfg, N, message_capacity=64)
        self.dpxa = rb.PaxosAcceptors(self.cfg, 1)
        self.dfp = rb.FastPaxos(self.cfg, N)
        self.checked = {k: 0 for k in ("fast2b", "1a", "1b", "2a", "2b")}

    def ids(self, tags):
        return [self.id_of_tag[t] for t in tags]

    def to_pb(self, kind, m):
        pb = self.pb
        k = {"fast2b": 5, "1a": 6, "1b": 7, "2a": 8, "2b": 9}[kind]
        x = pb.kind[k]()
        x.sender.hostname, x.sender.port = ep_of(self.id_of_tag[m["sender"]])
        x.configurationId = m["cfg"]
        if kind == "1a":
            x.rank.round, x.rank.nodeIndex = m["rank"]
        if kind in ("1b", "2a", "2b"):
            x.rnd.round, x.rnd.nodeIndex = m["rnd"]
        if kind == "1b":
            x.vrnd.round, x.vrnd.nodeIndex = m["vrnd"]
        for t in m.get("vval", m.get("endpoints", [])):
            getattr(x, WPC.LIST_NAME[k]).add(hostname=ep_of(self.id_of_tag[t])[0], port=ep_of(self.id_of_tag[t])[1])
        return k, pb.RapidRequest(**{WPC.CASES[k]: x}).SerializeToString()

    def send(self, i, kind, m):
        self.inbox[i].append((kind, m))
        if i == 0 and kind in ("fast2b", "2b") and self.rng.random() < 0.2:
            self.inbox[i].append((kind, m))                              # a duplicate sender
        if i == 0 and self.rng.random() < 0.1:
            self.inbox[i].append((kind, dict(m, cfg=m["cfg"] - 1)))      # a stale configuration

    def broadcast(self, kind, m):
        for i in range(self.N):
            self.send(i, kind, m)

    def propose(self, i, proposal):
        self.px[i].registerFastRoundVote(proposal)
        if i == 0:
            h1, h2 = self.rb.proposal_fingerprint(self.ids(proposal))
            self.dpxa.registerFastRoundVotes([0], [h1], [len(proposal)], [h2])
        self.broadcast("fast2b", {"sender": self.tags[i], "cfg": self.cfg, "endpoints": list(proposal)})

    def start(self, i, round_):
        m = self.px[i].startPhase1a(round_)
        if i == 0:
            assert self.dpx.startPhase1a(round_, self.hashes[0]) == (m is not None)
        if m:
            self.broadcast("1a", m)

    def deliver_other(self, i, kind, m):
        if kind == "fast2b":
            self.fp[i].handleFastRoundProposal(m["sender"], m["cfg"], m["endpoints"])
        elif kind == "1a":
            r = self.px[i].handlePhase1aMessage(m)
            if r:
                self.send(self.id_of_tag[m["sender"]], "1b", r)
        elif kind == "1b":
            r = self.px[i].handlePhase1bMessage(m)
            if r:
                self.broadcast("2a", r)
        elif kind == "2a":
            r = self.px[i].handlePhase2aMessage(m)
            if r:
                self.broadcast("2b", r)
        elif kind == "2b":
            self.px[i].handlePhase2bMessage(m)

    def deliver_node0(self, kind, batch):
        """the oracle one message at a time; the device the whole batch from bytes"""
        k_data = [self.to_pb(kind, m) for m in batch]
        k = k_data[0][0]
        self.dec.decodeConsensusMessages(k, [d for _, d in k_data], is_request=True)
        self.checked[kind] += len(batch)
        if kind == "fast2b":
            was = self.fp[0].decided()
            for m in batch:
                self.fp[0].handleFastRoundProposal(m["sender"], m["cfg"], m["endpoints"])
            r = self.dfp.handleFastRoundProposalsFromWire(self.dec)
            assert r.decided == self.fp[0].decided() and r.votes_received == self.fp[0].votesReceived()
            if r.decided and not was:
                assert (r.hash, r.hash2, r.length) == (*self.rb.proposal_fingerprint(self.ids(self.fp[0].decision())),
                                                       len(self.fp[0].decision()))
        elif kind in ("1a", "2a"):
            out = self.dec.consensusMessages()
            for i, m in enumerate(batch):                                # single broadcasts: the host reads the fields
                r = self.px[0].handlePhase1aMessage(m) if kind == "1a" else self.px[0].handlePhase2aMessage(m)
                rank = (int(out["rnd_round"][i]), int(out["rnd_node"][i]))
                if kind == "1a":
                    got = self.dpxa.handlePhase1aMessage(rank, msg_cfg=int(out["cfg"][i]))
                else:
                    got = self.dpxa.handlePhase2aMessage(rank, (int(out["hash"][i]), int(out["hash2"][i]), int(out["len"][i])),
                                                         msg_cfg=int(out["cfg"][i]))
                assert got == (1 if r else 0)
                if r and kind == "1a":
                    assert (r["vval"] and self.dpxa.read(0)["vval"][2] == len(r["vval"])) or not r["vval"]
                    self.send(self.id_of_tag[m["sender"]], "1b", r)
                elif r:
                    self.broadcast("2b", r)
        elif kind == "1b":
            trig = -1
            for i, m in enumerate(batch):
                r = self.px[0].handlePhase1bMessage(m)
                if r:
                    trig = i
                    self.broadcast("2a", r)
            got = self.dpx.handlePhase1bFromWire(self.dec)
            assert got.proposed == (trig >= 0) and got.trigger_index == trig
            if trig >= 0:                                                # cval: the value the coordinator rule chose
                cval = self.ids(self.px[0].cval())
                assert got.cval == (*self.rb.proposal_fingerprint(cval), len(cval))
                out = self.dec.consensusMessages()
                src = [i for i in range(len(batch)) if (int(out["hash"][i]), int(out["hash2"][i]), int(out["len"][i])) == got.cval]
                assert not src or self.dec.consensusValue(src[0]) == cval
        else:
            dec_at = -1
            for i, m in enumerate(batch):
                if self.px[0].handlePhase2bMessage(m) and dec_at < 0:
                    dec_at = i
            got = self.dpx.handlePhase2bFromWire(self.dec)
            assert got.decided == self.px[0].decided() and got.decided_index == dec_at
            if dec_at >= 0:
                assert self.ids(self.px[0].decision()) == self.dec.consensusValue(dec_at)

    def run(self):
        while True:
            ready = [i for i in range(self.N) if self.inbox[i]]
            if not ready:
                return
            i = self.rng.choice(ready)
            if i:
                self.deliver_other(i, *self.inbox[i].pop(0))
                continue
            kind = self.inbox[0][0][0]
            take = 1
            while take < len(self.inbox[0]) and self.inbox[0][take][0] == kind and take < self.rng.randint(1, 8):
                take += 1
            batch = [m for _, m in self.inbox[0][:take]]
            del self.inbox[0][:take]
            self.deliver_node0(kind, batch)


@pytest.mark.parametrize("N,seed", [(5, 1), (8, 2), (13, 3)])
def test_whole_rounds_against_the_oracle(orc, rb, pb, N, seed):
    net = WireNet(orc, rb, pb, N, seed)
    rng = random.Random(seed)
    a, b = sorted(rng.sample(net.tags, 2)), sorted(rng.sample(net.tags, 3))
    for i in range(N):                                                   # fast-round votes, split: the fast round cannot decide
        if rng.random() < 0.7:
            net.propose(i, a if i % 2 else b)
    net.run()
    for rnd, who in ((2, [0, 1]), (3, [N - 1, 0]), (4, [0])):           # several coordinators and rounds
        for i in who:
            net.start(i, rnd)
        net.run()
    assert all(v > 0 for v in net.checked.values()), net.checked
    assert net.px[0].decided()


# ------------------------------------------------------------------------------------------------ 7. refusals, stale votes
def test_unknown_senders_stale_votes_and_wrong_kinds(rb, pb):
    n, cfg = 16, 7
    view = make_view(rb, n)
    dec = rb.WireDecoder(view)
    val = [1, 2, 3]
    h = rb.proposal_fingerprint(val)

    def msg(kind, sender, c, rnd=(2, 1)):
        m = pb.kind[kind]()
        if sender is None:
            m.sender.hostname, m.sender.port = b"departed", 1
        else:
            m.sender.hostname, m.sender.port = ep_of(sender)
        m.configurationId = c
        if kind == WPC.PHASE2B:
            m.rnd.round, m.rnd.nodeIndex = rnd
        for j in val:
            getattr(m, WPC.LIST_NAME[kind]).add(hostname=ep_of(j)[0], port=ep_of(j)[1])
        return m.SerializeToString()

    # Phase2b: a current-configuration message of an unknown sender refuses, and the handle stays as a fresh one would
    good = [msg(9, s, cfg) for s in range(4)]
    a, b = rb.Paxos(cfg, n), rb.Paxos(cfg, n)
    dec.decodeConsensusMessages(9, good)
    a.handlePhase2bFromWire(dec); b.handlePhase2bFromWire(dec)
    dec.decodeConsensusMessages(9, [msg(9, 5, cfg), msg(9, None, cfg)])
    with pytest.raises(rb.RapidError, match="outside the dictionary"):
        a.handlePhase2bFromWire(dec)
    rest = [msg(9, s, cfg) for s in range(4, 10)]
    dec.decodeConsensusMessages(9, rest)
    ra, rb_ = a.handlePhase2bFromWire(dec), b.handlePhase2bFromWire(dec)
    assert (ra.decided, ra.decided_index, ra.decision) == (rb_.decided, rb_.decided_index, rb_.decision) and ra.decided
    # ... the same message with a stale configurationId is dropped, and the call decides as the Learner says
    p = rb.Paxos(cfg, n)
    stream = [msg(9, s, cfg) for s in range(5)] + [msg(9, None, cfg - 1)] + [msg(9, s, cfg) for s in range(5, 12)]
    dec.decodeConsensusMessages(9, stream)
    out = dec.consensusMessages()
    r = p.handlePhase2bFromWire(dec)
    L = plainref.Learner(n, cfg)
    want = L.handle(np.stack([out["rnd_round"], out["rnd_node"]], 1), out["sender"], out["hash"], out["len"], h2=out["hash2"],
                    msg_cfg=out["cfg"])
    assert (r.decided, r.decided_index, r.decision) == want and r.decided_index == 9 and r.decision == (h[0], h[1], 3)
    # the fast round: the same two rules (FastPaxos.java:126 drops a stale vote before anything else)
    votes = [msg(5, s, cfg) for s in range(6)]
    fa, fb = rb.FastPaxos(cfg, n), rb.FastPaxos(cfg, n)
    dec.decodeConsensusMessages(5, votes)
    fa.handleFastRoundProposalsFromWire(dec); fb.handleFastRoundProposalsFromWire(dec)
    dec.decodeConsensusMessages(5, [msg(5, 8, cfg), msg(5, None, cfg)])
    with pytest.raises(rb.RapidError, match="outside the dictionary"):
        fa.handleFastRoundProposalsFromWire(dec)
    stream = [msg(5, None, cfg - 1)] + [msg(5, s, cfg) for s in range(6, n)]
    dec.decodeConsensusMessages(5, stream)
    out = dec.consensusMessages()
    ra, rb_ = fa.handleFastRoundProposalsFromWire(dec), fb.handleFastRoundProposalsFromWire(dec)
    assert (ra.decided, ra.count, ra.votes_received) == (rb_.decided, rb_.count, rb_.votes_received)
    ref = plainref.FastRound(n)
    ref.call(list(range(6)), [h] * 6)
    keep = out["cfg"] == cfg
    ref.call(out["sender"][keep].tolist(), [h] * int(keep.sum()))
    assert (ra.decided, ra.count, ra.votes_received) == (ref.decided, ref.count, ref.votes_received) and ra.decided
    # Phase1b ignores its sender: an unknown one is not an error
    p = rb.Paxos(cfg, 4)
    p.startPhase1a(2, 1)
    m = pb.Phase1bMessage(configurationId=cfg)
    m.sender.hostname = b"departed"
    m.rnd.round, m.rnd.nodeIndex = 2, 1
    dec.decodeConsensusMessages(7, [m.SerializeToString()] * 3)
    assert p.handlePhase1bFromWire(dec).n_messages == 3
    # a wrong-kind decode, and a decode that was replaced by an alert decode, are refused
    with pytest.raises(rb.RapidError, match="Phase2bMessage"):
        p.handlePhase2bFromWire(dec)
    with pytest.raises(rb.RapidError, match="FastRoundPhase2bMessage"):
        fa.handleFastRoundProposalsFromWire(dec)
    dec.decodeBatchedAlertMessage(b"")
    with pytest.raises(rb.RapidError):
        p.handlePhase1bFromWire(dec)


def test_cross_device_refusal_needs_two_gpus(rb):
    """a px / fp on one device refuses a wire handle of another: this needs two GPUs"""
    from rapid_b200 import _native as N
    if N.device_count() < 2:
        pytest.skip("the cross-device refusal needs two GPUs; this machine has one")
    view = make_view(rb, 8)
    dec = rb.WireDecoder(view)
    dec.decodeConsensusMessages(5, [])
    fp = rb.FastPaxos(1, 8, device=1)
    with pytest.raises(rb.RapidError, match="different devices"):
        fp.handleFastRoundProposalsFromWire(dec)


# ------------------------------------------------------------------------------------------------ 8. scale and skew
def _enc_eps(n):
    hosts, ports = W.endpoints(0, n)
    return [WPC.enc_endpoint(h if isinstance(h, bytes) else h.encode(), int(p)) for h, p in zip(hosts, ports.tolist())]


def test_scale_phase1b_inbox_against_plainref(rb):
    Nview, n_msgs, N, cfg = 200_000, 100_000, 120_000, 4
    view = make_view(rb, Nview)
    eps = _enc_eps(Nview)
    rng = np.random.default_rng(3)
    values = [np.sort(rng.choice(Nview, 100, replace=False)).tolist() for _ in range(5)]
    lists = [WPC.enc_list(WPC.PHASE1B, [eps[j] for j in v]) for v in values]
    fps = [rb.proposal_fingerprint(v) for v in values]
    which = rng.integers(0, 5, n_msgs)
    vr_round = rng.integers(0, 3, n_msgs)
    senders = rng.integers(0, Nview, n_msgs)
    msgs = [WPC.enc_message(WPC.PHASE1B, eps[s], cfg, (2, 7), (int(r), 1), lists[w])
            for s, r, w in zip(senders.tolist(), vr_round.tolist(), which.tolist())]
    dec = rb.WireDecoder(view)
    assert dec.decodeConsensusMessages(WPC.PHASE1B, msgs) == (0, 0)
    ms = dec.lastDeviceMs()
    out = dec.consensusMessages()
    np.testing.assert_array_equal(out["sender"], senders)
    np.testing.assert_array_equal(out["vrnd_round"], vr_round)
    assert (out["len"] == 100).all() and (out["rnd_round"] == 2).all() and (out["rnd_node"] == 7).all()
    np.testing.assert_array_equal(out["hash"], np.array([fps[w][0] for w in which.tolist()], np.uint64))
    np.testing.assert_array_equal(out["hash2"], np.array([fps[w][1] for w in which.tolist()], np.uint64))
    px = rb.Paxos(cfg, N, message_capacity=n_msgs)
    px.startPhase1a(2, 7)
    r = px.handlePhase1bFromWire(dec)
    ref = plainref.Coordinator(N, cfg)
    ref.startPhase1a(2, 7)
    want = ref.handle(np.tile([2, 7], (n_msgs, 1)), np.stack([vr_round, np.ones(n_msgs, np.int64)], 1), out["hash"], out["len"],
                      h2=out["hash2"], msg_cfg=out["cfg"])
    assert (r.proposed, r.trigger_index, r.cval, r.n_messages) == want and r.proposed
    assert dec.consensusValue(r.trigger_index) == values[int(which[r.trigger_index])]
    print("Phase1b decode: %d messages x 100 endpoints, %.3f ms on the device" % (n_msgs, ms))


def test_one_huge_list_among_short_ones(rb):
    Nview = 60_000
    view = make_view(rb, Nview)
    eps = _enc_eps(Nview)
    rng = np.random.default_rng(4)
    big = rng.permutation(Nview)[:50_000].tolist()
    big[17] = -1                                                          # one stranger inside
    enc = lambda ids: WPC.enc_list(WPC.PHASE2B, [eps[j] if j >= 0 else WPC.enc_endpoint(b"nobody", 9) for j in ids])
    short = [rng.integers(0, Nview, 3).tolist() for _ in range(10_000)]
    msgs = [WPC.enc_message(WPC.PHASE2B, eps[i], 1, (2, 1), None, enc(s)) for i, s in enumerate(short)]
    at = 4321
    msgs.insert(at, WPC.enc_message(WPC.PHASE2B, eps[0], 1, (2, 1), None, enc(big)))
    dec = rb.WireDecoder(view)
    assert dec.decodeConsensusMessages(WPC.PHASE2B, msgs) == (0, 1)
    out = dec.consensusMessages()
    assert out["len"][at] == 50_000 and dec.consensusValue(at) == big
    known = [j for j in big if j >= 0]
    h1, h2 = rb.proposal_fingerprint(known)
    # the stranger's terms: what the vote decoder gives a one-stranger list
    dec2 = rb.WireDecoder(view)
    dec2.decodeConsensusMessages(WPC.FAST_ROUND_PHASE2B, [WPC.enc_list(5, [WPC.enc_endpoint(b"nobody", 9)])])
    o2 = dec2.consensusMessages()
    M = (1 << 64) - 1
    assert (int(out["hash"][at]), int(out["hash2"][at])) == ((h1 + int(o2["hash"][0])) & M, (h2 + int(o2["hash2"][0])) & M)
    for i in (0, at - 1, at + 1, len(msgs) - 1):
        s = short[i if i < at else i - 1]
        assert (int(out["hash"][i]), int(out["hash2"][i])) == rb.proposal_fingerprint(s) and dec.consensusValue(i) == s


def test_a_million_fast_round_votes(rb):
    N, cfg = 1_000_000, 9
    view = make_view(rb, N)
    eps = _enc_eps(N)
    rng = np.random.default_rng(5)
    va, vb = [1, 5, 9], [2, 5, 9]
    la, lb = WPC.enc_list(5, [eps[j] for j in va]), WPC.enc_list(5, [eps[j] for j in vb])
    pick_b = rng.random(N) < 0.08
    order = rng.permutation(N)
    hdr = WPC.varint(cfg)
    msgs = [b"\x0a" + WPC.varint(len(eps[s])) + eps[s] + b"\x10" + hdr + (lb if pb_ else la)
            for s, pb_ in zip(order.tolist(), pick_b[order].tolist())]
    dec = rb.WireDecoder(view)
    dec.decodeConsensusMessages(WPC.FAST_ROUND_PHASE2B, msgs)
    fp = rb.FastPaxos(cfg, N)
    r = fp.handleFastRoundProposalsFromWire(dec)
    fa, fbb = rb.proposal_fingerprint(va), rb.proposal_fingerprint(vb)
    ref = plainref.FastRound(N)
    ref.call(order.tolist(), [fbb if x else fa for x in pick_b[order].tolist()])
    assert ref.decided and ref.decided_at[1] < N - 1000
    assert (r.decided, (r.hash, r.hash2), r.count, r.votes_received) == (True, ref.decision, ref.count, ref.votes_received)
