"""CPU-side gates: the oracle against the committed golden fixtures, and the C-ABI library loads and exports every
symbol include/rapid_b200.h declares (no compute without a GPU; creation must fail loudly, never fall back)."""
import ctypes
import json
import os
import re

import numpy as np
import pytest

from rapid_b200 import workloads as W

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
K = 10


def _golden(name):
    with open(os.path.join(HERE, "golden", name)) as f:
        return json.load(f)


def test_oracle_matches_golden_ring_keys(orc):
    g = _golden("ring_keys.json")
    n = len(g["endpoints"])
    u = orc.Universe()
    tags = [u.add(e["hostname"], e["port"]) for e in g["endpoints"]]
    hi = [a for a, _ in g["node_ids"]]
    lo = [b for _, b in g["node_ids"]]
    v = orc.MembershipView(u, K, tags, hi, lo)
    for k in range(K):
        assert [v.key(k, i) for i in range(n)] == g["keys"][k]
        assert v.getRing(k) == g["rings"][k]
    assert v.getCurrentConfigurationId() == g["configuration_id"]
    assert orc.xxh64(b"", 0) == g["xxh64"]["empty_seed0"]
    assert orc.xx_hash_int(1000, 3) == g["xxh64"]["hashInt_1000_seed3"]
    assert orc.xx_hash_long(-1, 0) == g["xxh64"]["hashLong_minus1_seed0"]
    # the generator's own node-id rule
    ghi, glo = W.node_ids(0, n)
    assert ghi.tolist() == hi and glo.tolist() == lo


def test_oracle_matches_golden_cut_scenarios(orc):
    for c in _golden("cut_scenarios.json"):
        n, nj = c["n"], c["n_joiners"]
        hb, off, ports = W.packed_endpoints(0, n + nj)
        u = orc.Universe()
        tags = u.add_bulk(hb, off, ports)
        hi, lo = W.node_ids(0, n)
        v = orc.MembershipView(u, K, tags[:n], hi, lo)
        assert v.getCurrentConfigurationId() == c["configuration_id"]
        sim = orc.ClusterSim(v, K, c["H"], c["L"], n)
        blocked = np.zeros(n, np.uint8)
        blocked[c["blocked_receivers"]] = 1
        cells = c["cells"]
        o_len, o_ann, o_ids, o_off = sim.apply_batch(cells["src"], cells["dst"], cells["ring"], cells["status"],
                                                     np.full(len(cells["dst"]), c["configuration_id"], np.int64), blocked=blocked)
        assert sorted(set(o_len.tolist())) == c["proposal_len"]
        assert int(o_ann.sum()) == c["announced_count"]
        r0 = int(np.nonzero(o_len)[0][0])
        assert o_ids[o_off[r0]: o_off[r0 + 1]].tolist() == c["proposal_canonical"]
        assert sorted(c["proposal_canonical"]) == c["expected_cut"]


def test_oracle_matches_golden_paxos_rule_cases(orc):
    u = orc.Universe()
    vals = {0: []}
    for i in range(1, 6):
        vals[i] = [u.add("v", 10 * i + j) for j in range(1 + i % 3)]
    for c in _golden("paxos_rule_cases.json"):
        px = orc.ClassicPaxos(u, u.add("me", 1), 7, 1, c["N"])
        msgs = [{"vrnd": tuple(r), "vval": vals[v]} for r, v in zip(c["vrnd"], c["value"])]
        assert px.selectProposalUsingCoordinatorRule(msgs) == vals[c["chosen_value"]]


def test_oracle_matches_golden_failure_detector_stream(orc):
    g = _golden("failure_detector_stream.json")
    n, K = g["n"], g["K"]
    hb, off, ports = W.packed_endpoints(0, n)
    u = orc.Universe()
    tags = u.add_bulk(hb, off, ports)
    hi, lo = W.node_ids(0, n)
    sim = orc.FdSim(orc.MembershipView(u, K, tags, hi, lo), K, np.arange(n))
    flags = np.asarray(g["flags"], np.uint8)
    for want in g["intervals"]:
        assert [[o, s, r] for o, s, r in sim.tick(flags, g["cfg"])] == want
    assert sum(len(x) for x in g["intervals"]) > 0


def test_library_exports_every_declared_symbol():
    from rapid_b200 import _native, _build
    hdr = open(os.path.join(ROOT, "include", "rapid_b200.h")).read()
    declared = set(re.findall(r"\b(rapid_[a-z0-9_]+)\s*\(", hdr))
    declared.discard("rapid_delivery")
    assert len(declared) >= 40
    lib = ctypes.CDLL(_build.build_native())
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, missing
    # the Python binding knows every entry point it may call
    assert set(_native.SIGNATURES) | {"rapid_version"} <= declared
    assert "rapid_cd_debug_grid" in declared and "rapid_cd_debug_grid" in _native.SIGNATURES
    _native.lib()
    assert b"sm_90a" in _native.lib().rapid_version()


def test_no_cpu_fallback_without_a_device():
    import rapid_b200 as rb
    from rapid_b200 import _native
    if _native.device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(rb.RapidError) as e:
        rb.MembershipView(K, ["a", "b"], [1, 2])
    assert e.value.code == _native.ECUDA
    with pytest.raises(rb.RapidError):
        rb.FastPaxos(1, 10)
    for make in (lambda: rb.Paxos(1, 10), lambda: rb.PaxosAcceptors(1, 10)):      # the "next" rows fail just as loudly
        with pytest.raises(rb.RapidError) as e:
            make()
        assert e.value.code == _native.ECUDA


def test_product_never_touches_the_oracle():
    """the oracle is test infrastructure: nothing under rapid_b200/ may import, link or name it"""
    for dp, _, fs in os.walk(os.path.join(ROOT, "rapid_b200")):
        if "build" in dp:
            continue
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh")):
                src = open(os.path.join(dp, f)).read()
                assert "oracle" not in src.lower() or f == "workloads.py", (dp, f)


def test_workload_generators_are_deterministic(orc):
    """the synthetic scenarios are pure functions of (n, seed, ring topology): regenerate the golden cells"""
    for c in _golden("cut_scenarios.json"):
        n, nj = c["n"], c["n_joiners"]
        hb, off, ports = W.packed_endpoints(0, n + nj)
        u = orc.Universe()
        tags = u.add_bulk(hb, off, ports)
        hi, lo = W.node_ids(0, n)
        v = orc.MembershipView(u, K, tags[:n], hi, lo)
        obs = lambda ids: v.tables(ids)[0]
        if c["name"] == "c1":
            b = W.c1_single_crash(obs, n)
        elif c["name"] == "c2":
            b = W.c2_simultaneous_crash(obs, n, 0.01)
        elif c["name"] == "c3":
            b = W.c3_correlated_partition(obs, np.asarray(v.getRing(0)), n, 0.05)
        else:
            jo = np.asarray([v.getExpectedObserversOf(n + j) for j in range(nj)], np.int32)
            b = W.c5_churn(obs, jo, n, 3, nj)
        assert b.dst.tolist() == c["cells"]["dst"] and b.ring.tolist() == c["cells"]["ring"]
        assert b.src.tolist() == c["cells"]["src"] and b.status.tolist() == c["cells"]["status"]
        assert b.expected_cut.tolist() == c["expected_cut"]
        # a full table and a lookup callable give the same batch
        full_obs, _ = v.tables(np.arange(n, dtype=np.int32))
        b2 = W.c2_simultaneous_crash(full_obs, n, 0.01)
        b3 = W.c2_simultaneous_crash(obs, n, 0.01)
        assert b2.dst.tolist() == b3.dst.tolist() and b2.src.tolist() == b3.src.tolist()


def test_c4_stream_shape(orc):
    n = 500
    hb, off, ports = W.packed_endpoints(0, n)
    u = orc.Universe()
    tags = u.add_bulk(hb, off, ports)
    v = orc.MembershipView(u, K, tags, *W.node_ids(0, n))
    obs, _ = v.tables(np.arange(n, dtype=np.int32))
    bs = W.c4_flip_flop_stream(obs, n, 0.02, T=8)
    assert len(bs) == 8 and bs[-1].expected_cut is not None and all(b.expected_cut is None for b in bs[:-1])
    failed = set(bs[-1].expected_cut.tolist())
    seen = set()
    for b in bs:
        assert set(b.dst.tolist()) <= failed and not (set(b.src.tolist()) & failed)
        seen |= set(zip(b.dst.tolist(), b.ring.tolist()))
    # every report of every flapping node is sent at least once over the stream
    want = {(s, k) for s in failed for k in range(K) if int(obs[s, k]) not in failed}
    assert seen == want
    assert sum(len(b) for b in bs) > len(want)          # and some are re-sent (duplicates)
