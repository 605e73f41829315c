"""The hand encoders of wire_proto_consensus emit the protobuf runtime's bytes for every consensus message kind, bare and as
RapidRequest, so tests that need millions of messages can use them in place of the runtime (no GPU needed)."""
import random

import pytest

import wire_proto_consensus as WPC

KINDS = [WPC.FAST_ROUND_PHASE2B, WPC.PHASE1A, WPC.PHASE1B, WPC.PHASE2A, WPC.PHASE2B]


def _rank(rng):
    return (rng.choice([0, 1, -1, 2**31 - 1, -2**31, rng.randint(-2**31, 2**31 - 1)]),
            rng.choice([0, 5, -7, 2**31 - 1, -2**31]))


@pytest.mark.parametrize("kind", KINDS)
def test_hand_encoders_agree_with_the_runtime(kind):
    pb = WPC.build()
    rng = random.Random(kind)
    for _ in range(200):
        m = pb.kind[kind]()
        sender = None
        if rng.random() < 0.8:
            sender = (b"host-%d" % rng.randrange(50) if rng.random() < 0.9 else b"", rng.choice([0, 1, 65535, -3]))
            m.sender.hostname, m.sender.port = sender
        cfg = rng.choice([0, 1, -1, 2**63 - 1, -2**63, rng.getrandbits(40)])
        m.configurationId = cfg
        rnd = vrnd = None
        if WPC.RANK_NAME[kind] and rng.random() < 0.8:
            rnd = _rank(rng)
            r = getattr(m, WPC.RANK_NAME[kind]); r.round, r.nodeIndex = rnd
        if kind == WPC.PHASE1B and rng.random() < 0.8:
            vrnd = _rank(rng)
            m.vrnd.round, m.vrnd.nodeIndex = vrnd
        eps = []
        if WPC.LIST_NAME[kind]:
            for _ in range(rng.randint(0, 6)):
                e = (b"h%d" % rng.randrange(9), rng.randrange(3))
                getattr(m, WPC.LIST_NAME[kind]).add(hostname=e[0], port=e[1])
                eps.append(WPC.enc_endpoint(*e))
        mine = WPC.enc_message(kind, None if sender is None else WPC.enc_endpoint(*sender), cfg, rnd, vrnd,
                               WPC.enc_list(kind, eps) if eps else b"")
        assert mine == m.SerializeToString(deterministic=True)
        req = pb.RapidRequest(**{WPC.CASES[kind]: m}).SerializeToString(deterministic=True)
        assert WPC.enc_request(kind, mine) == req
