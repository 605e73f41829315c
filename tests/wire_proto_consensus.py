"""The consensus messages of rapid/src/main/proto/rapid.proto, built with the protobuf runtime from descriptors (there is no
protoc in the image): Endpoint :13-17, Rank :133-137, Phase1aMessage :139-144, Phase1bMessage :146-153, Phase2aMessage
:155-161, Phase2bMessage :163-169, FastRoundPhase2bMessage :124-129, and the RapidRequest oneof cases 4-9 (:21-35).
The runtime is the encoder AND the reference decoder the GPU decoder is compared with.  The hand encoders below emit exactly
the runtime's bytes (test_wire_proto_consensus_helpers.py checks that) and are used where millions of messages are needed."""
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

from wire_proto import field, varint

F = descriptor_pb2.FieldDescriptorProto

FAST_ROUND_PHASE2B, PHASE1A, PHASE1B, PHASE2A, PHASE2B = 5, 6, 7, 8, 9
NAMES = {FAST_ROUND_PHASE2B: "FastRoundPhase2bMessage", PHASE1A: "Phase1aMessage", PHASE1B: "Phase1bMessage",
         PHASE2A: "Phase2aMessage", PHASE2B: "Phase2bMessage"}
CASES = {FAST_ROUND_PHASE2B: "fastRoundPhase2bMessage", PHASE1A: "phase1aMessage", PHASE1B: "phase1bMessage",
         PHASE2A: "phase2aMessage", PHASE2B: "phase2bMessage"}
LIST_FIELD = {FAST_ROUND_PHASE2B: 3, PHASE1A: None, PHASE1B: 5, PHASE2A: 5, PHASE2B: 4}
LIST_NAME = {FAST_ROUND_PHASE2B: "endpoints", PHASE1A: None, PHASE1B: "vval", PHASE2A: "vval", PHASE2B: "endpoints"}
RANK_NAME = {FAST_ROUND_PHASE2B: None, PHASE1A: "rank", PHASE1B: "rnd", PHASE2A: "rnd", PHASE2B: "rnd"}


def _field(msg, name, number, ftype, label=F.LABEL_OPTIONAL, type_name=None, oneof=None):
    f = msg.field.add()
    f.name, f.number, f.type, f.label = name, number, ftype, label
    if type_name:
        f.type_name = type_name
    if oneof is not None:
        f.oneof_index = oneof
    return f


def build():
    fd = descriptor_pb2.FileDescriptorProto()
    fd.name, fd.package, fd.syntax = "rapid_wire_consensus_test.proto", "remoting", "proto3"
    m = fd.message_type.add(); m.name = "Endpoint"
    _field(m, "hostname", 1, F.TYPE_BYTES); _field(m, "port", 2, F.TYPE_INT32)
    m = fd.message_type.add(); m.name = "Rank"
    _field(m, "round", 1, F.TYPE_INT32); _field(m, "nodeIndex", 2, F.TYPE_INT32)
    ep, rank = ".remoting.Endpoint", ".remoting.Rank"
    m = fd.message_type.add(); m.name = "FastRoundPhase2bMessage"
    _field(m, "sender", 1, F.TYPE_MESSAGE, type_name=ep); _field(m, "configurationId", 2, F.TYPE_INT64)
    _field(m, "endpoints", 3, F.TYPE_MESSAGE, F.LABEL_REPEATED, ep)
    m = fd.message_type.add(); m.name = "Phase1aMessage"
    _field(m, "sender", 1, F.TYPE_MESSAGE, type_name=ep); _field(m, "configurationId", 2, F.TYPE_INT64)
    _field(m, "rank", 3, F.TYPE_MESSAGE, type_name=rank)
    m = fd.message_type.add(); m.name = "Phase1bMessage"
    _field(m, "sender", 1, F.TYPE_MESSAGE, type_name=ep); _field(m, "configurationId", 2, F.TYPE_INT64)
    _field(m, "rnd", 3, F.TYPE_MESSAGE, type_name=rank); _field(m, "vrnd", 4, F.TYPE_MESSAGE, type_name=rank)
    _field(m, "vval", 5, F.TYPE_MESSAGE, F.LABEL_REPEATED, ep)
    m = fd.message_type.add(); m.name = "Phase2aMessage"
    _field(m, "sender", 1, F.TYPE_MESSAGE, type_name=ep); _field(m, "configurationId", 2, F.TYPE_INT64)
    _field(m, "rnd", 3, F.TYPE_MESSAGE, type_name=rank); _field(m, "vval", 5, F.TYPE_MESSAGE, F.LABEL_REPEATED, ep)
    m = fd.message_type.add(); m.name = "Phase2bMessage"
    _field(m, "sender", 1, F.TYPE_MESSAGE, type_name=ep); _field(m, "configurationId", 2, F.TYPE_INT64)
    _field(m, "rnd", 3, F.TYPE_MESSAGE, type_name=rank); _field(m, "endpoints", 4, F.TYPE_MESSAGE, F.LABEL_REPEATED, ep)
    m = fd.message_type.add(); m.name = "ProbeMessage"
    _field(m, "sender", 1, F.TYPE_MESSAGE, type_name=ep)
    m = fd.message_type.add(); m.name = "RapidRequest"
    m.oneof_decl.add().name = "content"
    _field(m, "probeMessage", 4, F.TYPE_MESSAGE, type_name=".remoting.ProbeMessage", oneof=0)
    for kind in (FAST_ROUND_PHASE2B, PHASE1A, PHASE1B, PHASE2A, PHASE2B):
        _field(m, CASES[kind], kind, F.TYPE_MESSAGE, type_name=".remoting." + NAMES[kind], oneof=0)
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)

    class NS:
        pass
    ns = NS()
    for name in ["Endpoint", "Rank", "ProbeMessage", "RapidRequest"] + list(NAMES.values()):
        setattr(ns, name, message_factory.GetMessageClass(pool.FindMessageTypeByName("remoting." + name)))
    ns.kind = {k: getattr(ns, v) for k, v in NAMES.items()}
    return ns


# ---------------------------------------------------------------- hand encoders (the runtime's canonical bytes)
def enc_endpoint(hostname, port):
    """an Endpoint's payload: proto3 omits default-valued fields"""
    h = hostname.encode() if isinstance(hostname, str) else bytes(hostname)
    return (field(1, 2, h) if h else b"") + (field(2, 0, varint(port)) if port else b"")


def enc_rank(rank):
    r, i = rank
    return (field(1, 0, varint(r)) if r else b"") + (field(2, 0, varint(i)) if i else b"")


def enc_message(kind, sender=None, cfg=0, rnd=None, vrnd=None, endpoint_fields=b""):
    """message `kind`; sender: Endpoint payload or None (absent); rnd / vrnd: (round, node) or None (absent);
    endpoint_fields: the list, already encoded as repeated fields (see enc_list)"""
    out = b""
    if sender is not None:
        out += field(1, 2, sender)
    if cfg:
        out += field(2, 0, varint(cfg))
    if rnd is not None:
        out += field(3, 2, enc_rank(rnd))
    if vrnd is not None:
        out += field(4, 2, enc_rank(vrnd))
    return out + endpoint_fields


def enc_list(kind, endpoint_payloads):
    f = LIST_FIELD[kind]
    return b"".join(field(f, 2, e) for e in endpoint_payloads)


def enc_request(kind, payload):
    return field(kind, 2, payload)
