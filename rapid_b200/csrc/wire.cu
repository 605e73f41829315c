// Wire-format ingest (SURVEY.md §8 f3): serialized protobuf (rapid.proto) -> cell SoA + Endpoint -> id, on the device.
//
// The host only walks the TOP level of a BatchedAlertMessage (one tag + one length per AlertMessage) to find the
// submessage ranges; everything inside them — varints, nested Endpoints, packed / unpacked ring numbers, NodeId,
// unknown fields — is parsed by one thread per AlertMessage.  Endpoints are resolved against an open-addressing
// table over the view's endpoints keyed by the ring-0 key the view already holds (MembershipView.java:579-582),
// with a byte compare on a hit.  Two passes over the messages: parse + count ring numbers, prefix sum, emit cells.
// Consensus messages (FastRoundPhase2b, Phase1a/1b/2a/2b) go through one load-balanced decoder: a thread per message for the
// top level, a scan over the list lengths, a thread per list ENTRY for the lookups, a warp per message for the fingerprint.
#include <limits.h>

#include <algorithm>
#include <map>
#include <string>
#include <utility>
#include <vector>


#include "common.cuh"
#include "scan.cuh"
#include "wire_internal.cuh"

namespace rapid {

// ------------------------------------------------------------------ protobuf wire primitives (host + device)
struct Rd {
    const uint8_t* p;
    const uint8_t* end;
    bool ok;
};
RAPID_HD uint64_t rd_varint(Rd& r) {
    uint64_t v = 0;
    for (int shift = 0; shift < 70; shift += 7) {
        if (r.p >= r.end) break;
        const uint8_t b = *r.p++;
        if (shift < 64) v |= (uint64_t)(b & 0x7f) << shift;
        if (!(b & 0x80)) return v;
    }
    r.ok = false;                       // truncated, or longer than 10 bytes
    return 0;
}
// after a tag: the payload range of a length-delimited field
RAPID_HD bool rd_len(Rd& r, const uint8_t** p, int64_t* len) {
    const uint64_t n = rd_varint(r);
    if (!r.ok || n > (uint64_t)(r.end - r.p)) { r.ok = false; return false; }
    *p = r.p; *len = (int64_t)n;
    r.p += n;
    return true;
}
RAPID_HD void rd_skip(Rd& r, uint32_t wire_type) {
    switch (wire_type) {
        case 0: rd_varint(r); break;
        case 1: if (r.end - r.p < 8) r.ok = false; else r.p += 8; break;
        case 2: { const uint8_t* p; int64_t n; rd_len(r, &p, &n); break; }
        case 5: if (r.end - r.p < 4) r.ok = false; else r.p += 4; break;
        default: r.ok = false;          // groups are not used by rapid.proto
    }
}

struct EpRef {                          // an Endpoint as it sits in the input buffer (rapid.proto:13-17)
    int32_t off, len, port, present;
};
// parse (merge) one Endpoint occurrence
RAPID_HD void parse_endpoint(const uint8_t* base, const uint8_t* p, int64_t n, EpRef* e, bool* ok) {
    Rd r{p, p + n, true};
    e->present = 1;
    while (r.ok && r.p < r.end) {
        const uint64_t tag = rd_varint(r);
        if (!r.ok) break;
        const uint32_t f = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
        if (f == 1 && wt == 2) { const uint8_t* q; int64_t l; if (rd_len(r, &q, &l)) { e->off = (int32_t)(q - base); e->len = (int32_t)l; } }
        else if (f == 2 && wt == 0) e->port = (int32_t)rd_varint(r);
        else if (f == 0) r.ok = false;
        else rd_skip(r, wt);
    }
    if (!r.ok) *ok = false;
}

struct MsgRec {                         // one AlertMessage (rapid.proto:101-110)
    EpRef src, dst;
    int64_t cfg, nid_high, nid_low;
    int32_t status, n_rings, has_nid, meta_off, meta_len, src_id, dst_id, pad_;
};

// ------------------------------------------------------------------ endpoint dictionary
__device__ __forceinline__ uint32_t ep_slot(int64_t key0) { return (uint32_t)(splitmix64((uint64_t)key0) >> 32); }

__global__ void k_wire_table_build(int64_t tot, const int64_t* __restrict__ key0, uint32_t T, int32_t* __restrict__ table) {
    const int64_t id = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= tot) return;
    uint32_t pos = ep_slot(key0[id]) & (T - 1);
    for (;;) {
        if (atomicCAS(&table[pos], -1, (int32_t)id) == -1) return;
        pos = (pos + 1) & (T - 1);
    }
}

// id of the endpoint e whose ring-0 key is k, -1 if the dictionary does not hold it
__device__ int32_t ep_lookup_key(const uint8_t* __restrict__ buf, const EpRef e, int64_t k, uint32_t T, const int32_t* __restrict__ table,
                                 const int64_t* __restrict__ key0, const uint8_t* __restrict__ hb, const int32_t* __restrict__ hoff,
                                 const int32_t* __restrict__ hport) {
    uint32_t pos = ep_slot(k) & (T - 1);
    for (uint32_t probes = 0; probes < T; ++probes) {
        const int32_t id = table[pos];
        if (id < 0) return -1;
        if (key0[id] == k && hport[id] == e.port && hoff[id + 1] - hoff[id] == e.len) {
            const uint8_t* a = hb + hoff[id];
            const uint8_t* b = buf + e.off;
            bool same = true;
            for (int32_t i = 0; i < e.len; ++i) if (a[i] != b[i]) { same = false; break; }
            if (same) return id;
        }
        pos = (pos + 1) & (T - 1);
    }
    return -1;
}
__device__ int32_t ep_lookup(const uint8_t* __restrict__ buf, const EpRef e, uint32_t T, const int32_t* __restrict__ table,
                             const int64_t* __restrict__ key0, const uint8_t* __restrict__ hb, const int32_t* __restrict__ hoff,
                             const int32_t* __restrict__ hport) {
    if (!e.present) return -1;
    return ep_lookup_key(buf, e, ring_key(buf + e.off, e.len, e.port, 0), T, table, key0, hb, hoff, hport);
}

struct Dict {
    uint32_t T;
    const int32_t* table;
    const int64_t* key0;
    const uint8_t* hb;
    const int32_t* hoff;
    const int32_t* hport;
};

struct WireScal {
    int32_t bad_msg;        // lowest index of a malformed message, INT_MAX if none
    int32_t n_need;         // UP alerts whose edgeDst is not in the dictionary
    int32_t n_cells, n_dropped, sender_id;
    int32_t n_items;        // consensus decode: endpoints in all the lists
    int32_t n_unknown_senders, n_unknown_endpoints;
};

// ------------------------------------------------------------------ alert kernels
// pass 1: parse every AlertMessage, resolve its endpoints, count its ring numbers
__global__ void k_wire_parse_alerts(int64_t M, const uint8_t* __restrict__ buf, const int64_t* __restrict__ moff,
                                    const int32_t* __restrict__ mlen, Dict d, MsgRec* __restrict__ rec, int32_t* __restrict__ need,
                                    WireScal* __restrict__ sc, int have_cfg, int64_t cur_cfg) {
    const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    MsgRec r;
    memset(&r, 0, sizeof(r));
    const uint8_t* p0 = buf + moff[m];
    Rd rd{p0, p0 + mlen[m], true};
    bool ok = true;
    while (rd.ok && rd.p < rd.end) {
        const uint64_t tag = rd_varint(rd);
        if (!rd.ok) break;
        const uint32_t f = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
        const uint8_t* q; int64_t l;
        if (f == 1 && wt == 2) { if (rd_len(rd, &q, &l)) parse_endpoint(buf, q, l, &r.src, &ok); }
        else if (f == 2 && wt == 2) { if (rd_len(rd, &q, &l)) parse_endpoint(buf, q, l, &r.dst, &ok); }
        else if (f == 3 && wt == 0) r.status = (int32_t)rd_varint(rd);
        else if (f == 4 && wt == 0) r.cfg = (int64_t)rd_varint(rd);
        else if (f == 5 && wt == 0) { rd_varint(rd); ++r.n_rings; }                       // unpacked repeated int32
        else if (f == 5 && wt == 2) {                                                     // packed
            if (rd_len(rd, &q, &l)) { Rd pr{q, q + l, true}; while (pr.ok && pr.p < pr.end) { rd_varint(pr); ++r.n_rings; } if (!pr.ok) ok = false; }
        }
        else if (f == 6 && wt == 2) {                                                     // NodeId {high = 1, low = 2}
            if (rd_len(rd, &q, &l)) {
                r.has_nid = 1;
                Rd nr{q, q + l, true};
                while (nr.ok && nr.p < nr.end) {
                    const uint64_t t2 = rd_varint(nr);
                    if (!nr.ok) break;
                    if ((t2 >> 3) == 1 && (t2 & 7) == 0) r.nid_high = (int64_t)rd_varint(nr);
                    else if ((t2 >> 3) == 2 && (t2 & 7) == 0) r.nid_low = (int64_t)rd_varint(nr);
                    else if ((t2 >> 3) == 0) nr.ok = false;
                    else rd_skip(nr, (uint32_t)(t2 & 7));
                }
                if (!nr.ok) ok = false;
            }
        }
        else if (f == 7 && wt == 2) { if (rd_len(rd, &q, &l)) { r.meta_off = (int32_t)(q - buf); r.meta_len = (int32_t)l; } }
        else if (f == 0) rd.ok = false;
        else rd_skip(rd, wt);
    }
    if (!rd.ok || !ok || r.status < 0 || r.status > 1) { atomicMin(&sc->bad_msg, (int32_t)m); r.n_rings = 0; r.src.present = r.dst.present = 0; }
    r.src_id = ep_lookup(buf, r.src, d.T, d.table, d.key0, d.hb, d.hoff, d.hport);
    r.dst_id = r.dst.present ? ep_lookup(buf, r.dst, d.T, d.table, d.key0, d.hb, d.hoff, d.hport) : -1;
    // a default-valued edgeDst (field absent) is the endpoint {"" , 0}: resolvable like any other
    if (!r.dst.present) { EpRef e{0, 0, 0, 1}; r.dst = e; r.dst_id = ep_lookup(buf, e, d.T, d.table, d.key0, d.hb, d.hoff, d.hport); }
    // UP about an unknown endpoint: a joiner — but only an alert of the CURRENT configuration may introduce one (a stale one is
    // dropped by filterAlertMessages, MembershipService.java:653, before extractJoinerUuidAndMetadata ever sees it)
    const bool nd = r.dst_id < 0 && r.status == 0 && (!have_cfg || r.cfg == cur_cfg);
    need[m] = nd ? 1 : 0;
    if (nd) atomicAdd(&sc->n_need, 1);
    rec[m] = r;
}
// after joiners were registered: resolve what was unknown
__global__ void k_wire_relookup(int64_t M, const uint8_t* __restrict__ buf, Dict d, MsgRec* __restrict__ rec) {
    const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    if (rec[m].dst_id < 0) rec[m].dst_id = ep_lookup(buf, rec[m].dst, d.T, d.table, d.key0, d.hb, d.hoff, d.hport);
    if (rec[m].src_id < 0) rec[m].src_id = ep_lookup(buf, rec[m].src, d.T, d.table, d.key0, d.hb, d.hoff, d.hport);
}
__global__ void k_wire_counts(int64_t M, const MsgRec* __restrict__ rec, int32_t* __restrict__ cnt, WireScal* __restrict__ sc) {
    const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    const bool drop = rec[m].dst_id < 0;
    cnt[m] = drop ? 0 : rec[m].n_rings;
    if (drop) atomicAdd(&sc->n_dropped, 1);
}
// pass 2: one cell per ring number, in message order then ring order
__global__ void k_wire_emit(int64_t M, const uint8_t* __restrict__ buf, const int64_t* __restrict__ moff, const int32_t* __restrict__ mlen,
                            const MsgRec* __restrict__ rec, const int32_t* __restrict__ cnt, const int32_t* __restrict__ pos,
                            int32_t* __restrict__ o_src, int32_t* __restrict__ o_dst, uint8_t* __restrict__ o_ring,
                            uint8_t* __restrict__ o_status, int64_t* __restrict__ o_cfg, WireScal* __restrict__ sc) {
    const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    if (m == M - 1) sc->n_cells = pos[m] + cnt[m];
    if (cnt[m] == 0) return;
    const MsgRec r = rec[m];
    int32_t j = pos[m];
    const uint8_t* p0 = buf + moff[m];
    Rd rd{p0, p0 + mlen[m], true};
    while (rd.ok && rd.p < rd.end) {
        const uint64_t tag = rd_varint(rd);
        if (!rd.ok) break;
        const uint32_t f = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
        if (f == 5 && wt == 0) {
            const int32_t ring = (int32_t)rd_varint(rd);
            o_src[j] = r.src_id; o_dst[j] = r.dst_id; o_ring[j] = (uint8_t)(ring < 0 || ring > 255 ? 255 : ring);
            o_status[j] = (uint8_t)r.status; o_cfg[j] = r.cfg; ++j;
        } else if (f == 5 && wt == 2) {
            const uint8_t* q; int64_t l;
            if (rd_len(rd, &q, &l)) {
                Rd pr{q, q + l, true};
                while (pr.ok && pr.p < pr.end) {
                    const int32_t ring = (int32_t)rd_varint(pr);
                    o_src[j] = r.src_id; o_dst[j] = r.dst_id; o_ring[j] = (uint8_t)(ring < 0 || ring > 255 ? 255 : ring);
                    o_status[j] = (uint8_t)r.status; o_cfg[j] = r.cfg; ++j;
                }
            }
        } else rd_skip(rd, wt);
    }
}
__global__ void k_wire_begin(WireScal* sc) {
    sc->bad_msg = INT_MAX; sc->n_need = 0; sc->n_cells = 0; sc->n_dropped = 0; sc->sender_id = -1;
    sc->n_items = 0; sc->n_unknown_senders = 0; sc->n_unknown_endpoints = 0;
}
__global__ void k_wire_sender(const uint8_t* __restrict__ buf, EpRef e, Dict d, WireScal* __restrict__ sc) {
    sc->sender_id = ep_lookup(buf, e, d.T, d.table, d.key0, d.hb, d.hoff, d.hport);
}
__global__ void k_wire_msg_fields(int64_t M, const MsgRec* __restrict__ rec, int32_t* dst, uint8_t* status, int32_t* n_rings, int64_t* nh,
                                  int64_t* nl, uint8_t* has, int64_t* moff, int32_t* mlen) {
    const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    const MsgRec r = rec[m];
    dst[m] = r.dst_id; status[m] = (uint8_t)r.status; n_rings[m] = r.n_rings; nh[m] = r.nid_high; nl[m] = r.nid_low;
    has[m] = (uint8_t)r.has_nid; moff[m] = r.meta_off; mlen[m] = r.meta_len;
}

// ------------------------------------------------------------------ consensus messages (rapid.proto:124-169)
// Kinds are the RapidRequest oneof cases (rapid.proto:21-35).  Every kind is {sender = 1, configurationId = 2} plus up to two
// Ranks and one repeated Endpoint list; the layout says which field numbers carry them (0: none).
struct ConsLayout {
    uint32_t rank_a;        // rank (Phase1a) or rnd
    uint32_t rank_b;        // vrnd (Phase1b)
    uint32_t list;          // endpoints / vval
};
RAPID_HD ConsLayout cons_layout(int32_t kind) {
    switch (kind) {
        case RAPID_WIRE_FAST_ROUND_PHASE2B: return ConsLayout{0, 0, 3};
        case RAPID_WIRE_PHASE1A: return ConsLayout{3, 0, 0};
        case RAPID_WIRE_PHASE1B: return ConsLayout{3, 4, 5};
        case RAPID_WIRE_PHASE2A: return ConsLayout{3, 0, 5};
        default: return ConsLayout{3, 0, 4};                 // RAPID_WIRE_PHASE2B: its list is field 4
    }
}

// parse (merge) one Rank occurrence {round = 1, nodeIndex = 2}: int32 fields are the low 32 bits of the varint
RAPID_HD void parse_rank(const uint8_t* p, int64_t n, int32_t* round, int32_t* node, bool* ok) {
    Rd r{p, p + n, true};
    while (r.ok && r.p < r.end) {
        const uint64_t tag = rd_varint(r);
        if (!r.ok) break;
        const uint32_t f = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
        if (f == 0) r.ok = false;
        else if (f == 1 && wt == 0) *round = (int32_t)rd_varint(r);
        else if (f == 2 && wt == 0) *node = (int32_t)rd_varint(r);
        else rd_skip(r, wt);
    }
    if (!r.ok) *ok = false;
}

struct ConsTop {                        // the top-level fields of one message
    EpRef sender;
    int64_t cfg;
    int32_t ra_round, ra_node, rb_round, rb_node;
    int32_t cnt;                        // list endpoints
    bool ok;
};

// Walk one occurrence of the message's content.  EMIT = false: parse everything but the list entries, count those.
// EMIT = true (the message is known to be well-formed): write the byte range and message index of every list entry.
template <bool EMIT>
__device__ void cons_part(const uint8_t* buf, const uint8_t* p, int64_t l, const ConsLayout L, ConsTop& t, int32_t msg,
                          int32_t* o_off, int32_t* o_len, int32_t* o_msg) {
    Rd r{p, p + l, true};
    while (r.ok && r.p < r.end) {
        const uint64_t tag = rd_varint(r);
        if (!r.ok) break;
        const uint32_t f = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
        const uint8_t* q; int64_t ql;
        if (f == 0) r.ok = false;
        else if (f == L.list && wt == 2) {
            if (rd_len(r, &q, &ql)) {
                if (EMIT) { o_off[t.cnt] = (int32_t)(q - buf); o_len[t.cnt] = (int32_t)ql; o_msg[t.cnt] = msg; }
                ++t.cnt;
            }
        }
        else if (EMIT) rd_skip(r, wt);
        else if (f == 1 && wt == 2) { if (rd_len(r, &q, &ql)) parse_endpoint(buf, q, ql, &t.sender, &t.ok); }
        else if (f == 2 && wt == 0) t.cfg = (int64_t)rd_varint(r);
        else if (f == L.rank_a && wt == 2) { if (rd_len(r, &q, &ql)) parse_rank(q, ql, &t.ra_round, &t.ra_node, &t.ok); }
        else if (f == L.rank_b && wt == 2) { if (rd_len(r, &q, &ql)) parse_rank(q, ql, &t.rb_round, &t.rb_node, &t.ok); }
        else rd_skip(r, wt);                                // unknown field, or a known one with another wire type
    }
    if (!r.ok) t.ok = false;
}

// Walk the message content of bytes [p, p + l): the whole range, or (unwrap) the RapidRequest's `kind` case.  A oneof case of
// message type that occurs several times is merged (the occurrences are walked in order into the same ConsTop); another case
// occurring later replaces it.  false: malformed RapidRequest, or its content is not (or no longer) the `kind` case.
template <bool EMIT>
__device__ bool cons_walk(const uint8_t* buf, const uint8_t* p, int64_t l, bool unwrap, int32_t kind, const ConsLayout L, ConsTop& t,
                          int32_t msg, int32_t* o_off, int32_t* o_len, int32_t* o_msg) {
    if (!unwrap) { cons_part<EMIT>(buf, p, l, L, t, msg, o_off, o_len, o_msg); return true; }
    Rd r{p, p + l, true};
    const uint8_t* from = p;
    bool have = false;
    while (r.ok && r.p < r.end) {
        const uint64_t tag = rd_varint(r);
        if (!r.ok) break;
        const uint32_t f = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
        if (f == 0) { r.ok = false; break; }
        if (wt == 2 && f <= 10) {                           // a case of RapidRequest.content (all are messages)
            const uint8_t* q; int64_t ql;
            if (!rd_len(r, &q, &ql)) break;
            if ((int32_t)f == kind) have = true;
            else { have = false; from = r.p; }
        } else rd_skip(r, wt);
    }
    if (!r.ok || !have) return false;
    Rd r2{from, p + l, true};
    while (r2.p < r2.end) {
        const uint64_t tag = rd_varint(r2);
        const uint32_t f = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
        const uint8_t* q; int64_t ql;
        if (wt == 2 && (int32_t)f == kind) { rd_len(r2, &q, &ql); cons_part<EMIT>(buf, q, ql, L, t, msg, o_off, o_len, o_msg); }
        else rd_skip(r2, wt);
    }
    return true;
}

// The one routine that turns a list endpoint into its terms of the order-insensitive list fingerprint: the id's mixes, as
// rapid_proposal_fingerprint sums them, or for an endpoint outside the dictionary (a delayed message of another configuration
// naming a node that has since left, say) mixes of its ring-0 key k.  So a list keeps one fingerprint whichever kind carries it,
// identical stranger lists keep identical fingerprints, and the tallies' configuration filters decide what the message is worth.
__device__ __forceinline__ void ep_fp_terms(int32_t id, int64_t k, uint64_t* a, uint64_t* b) {
    if (id >= 0) { *a = fp_mix1(id); *b = fp_mix2(id); return; }
    const uint64_t kk = (uint64_t)k;
    *a = splitmix64(kk ^ 0x554E4B4E4F574E31ULL);
    *b = splitmix64((kk * 0xD6E8FEB86659FD93ULL) ^ 0x554E4B4E4F574E32ULL);
}

// step 1, one thread per message: unwrap, top-level walk, sender lookup, list length
__global__ void k_cons_top(int64_t n, const uint8_t* __restrict__ buf, const int64_t* __restrict__ off, int unwrap, int32_t kind, Dict d,
                           int32_t* __restrict__ sender, int64_t* __restrict__ cfg, int32_t* __restrict__ ra_round,
                           int32_t* __restrict__ ra_node, int32_t* __restrict__ rb_round, int32_t* __restrict__ rb_node,
                           int32_t* __restrict__ cnt, WireScal* __restrict__ sc) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool unknown = false;
    if (i < n) {
        ConsTop t;
        memset(&t, 0, sizeof(t));
        t.ok = true;
        const int64_t l = off[i + 1] - off[i];
        const bool ok = cons_walk<false>(buf, buf + off[i], l, unwrap != 0, kind, cons_layout(kind), t, 0, nullptr, nullptr, nullptr) && t.ok;
        if (!ok) {
            atomicMin(&sc->bad_msg, (int32_t)i);
            memset(&t, 0, sizeof(t));
        }
        const int32_t s = ok ? ep_lookup(buf, t.sender, d.T, d.table, d.key0, d.hb, d.hoff, d.hport) : -1;
        unknown = ok && s < 0;
        sender[i] = s; cfg[i] = t.cfg;
        ra_round[i] = t.ra_round; ra_node[i] = t.ra_node; rb_round[i] = t.rb_round; rb_node[i] = t.rb_node;
        cnt[i] = t.cnt;
    }
    const unsigned u = __ballot_sync(0xffffffffu, unknown);
    if ((threadIdx.x & 31) == 0 && u) atomicAdd(&sc->n_unknown_senders, __popc(u));
}

// step 3, one thread per message: the byte range of every list entry, at its message's offset of the flat array
__global__ void k_cons_items(int64_t n, const uint8_t* __restrict__ buf, const int64_t* __restrict__ off, int unwrap, int32_t kind,
                             const int32_t* __restrict__ cnt, const int32_t* __restrict__ pos, int32_t* __restrict__ i_off,
                             int32_t* __restrict__ i_len, int32_t* __restrict__ i_msg) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || cnt[i] == 0) return;
    ConsTop t;
    memset(&t, 0, sizeof(t));
    const int32_t b = pos[i];
    cons_walk<true>(buf, buf + off[i], off[i + 1] - off[i], unwrap != 0, kind, cons_layout(kind), t, (int32_t)i, i_off + b, i_len + b,
                    i_msg + b);
}

// step 4, one thread per list entry: parse, look up, fingerprint terms
__global__ void k_cons_resolve(int64_t m, const uint8_t* __restrict__ buf, const int32_t* __restrict__ i_off,
                               const int32_t* __restrict__ i_len, const int32_t* __restrict__ i_msg, Dict d, int32_t* __restrict__ ids,
                               uint64_t* __restrict__ m1, uint64_t* __restrict__ m2, WireScal* __restrict__ sc) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool unknown = false;
    if (j < m) {
        EpRef e{0, 0, 0, 0};
        bool ok = true;
        parse_endpoint(buf, buf + i_off[j], i_len[j], &e, &ok);
        if (!ok) atomicMin(&sc->bad_msg, i_msg[j]);
        const int64_t k = ring_key(buf + e.off, e.len, e.port, 0);
        const int32_t id = ep_lookup_key(buf, e, k, d.T, d.table, d.key0, d.hb, d.hoff, d.hport);
        uint64_t a, b;
        ep_fp_terms(id, k, &a, &b);
        ids[j] = id; m1[j] = a; m2[j] = b;
        unknown = id < 0;
    }
    const unsigned u = __ballot_sync(0xffffffffu, unknown);
    if ((threadIdx.x & 31) == 0 && u) atomicAdd(&sc->n_unknown_endpoints, __popc(u));
}

// step 5, one warp per message: segmented sum of the terms (lane-strided, then shuffles)
__global__ void k_cons_reduce(int64_t n, const int32_t* __restrict__ pos, const int32_t* __restrict__ cnt, const uint64_t* __restrict__ m1,
                              const uint64_t* __restrict__ m2, uint64_t* __restrict__ h1, uint64_t* __restrict__ h2) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n) return;                                     // uniform across the warp
    const int32_t b = pos[i], c = cnt[i];
    uint64_t a = 0, e = 0;
    for (int32_t q = lane; q < c; q += 32) { a += m1[b + q]; e += m2[b + q]; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); e += __shfl_xor_sync(0xffffffffu, e, o); }
    if (lane == 0) { h1[i] = a; h2[i] = e; }
}

// ------------------------------------------------------------------ handle
struct Wire {
    rapid_view* view = nullptr;
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    float last_ms = 0.f;
    uint64_t table_epoch = 0;
    bool have_cfg = false;            // rapid_wire_set_configuration: only alerts of this configuration register joiners
    int64_t cur_cfg = 0;
    uint32_t T = 0;
    DevBuf<int32_t> table;
    DevBuf<uint8_t> buf;
    DevBuf<int64_t> moff;
    DevBuf<int32_t> mlen, need, cnt, pos, scan_sums;
    DevBuf<MsgRec> rec;
    DevBuf<WireScal> sc;
    PinnedBuf<WireScal> h_sc;
    int64_t M = 0, n_cells = 0;
    DevBuf<int32_t> o_src, o_dst;
    DevBuf<uint8_t> o_ring, o_status;
    DevBuf<int64_t> o_cfg;
    // message-field staging
    DevBuf<int64_t> t_i64a, t_i64b, t_i64c;
    DevBuf<int32_t> t_i32a, t_i32b, t_i32c;
    DevBuf<uint8_t> t_u8a, t_u8b;
    // the last consensus decode: per message (c_*), then per list entry in message order (i_*)
    int32_t cons_kind = 0;            // its kind; 0 if the last decode was not a consensus decode or was refused
    int64_t cons_n = 0;
    DevBuf<int64_t> c_off, c_cfg;
    DevBuf<int32_t> c_sender, c_ra_round, c_ra_node, c_rb_round, c_rb_node, c_len, c_pos;
    DevBuf<uint64_t> c_h1, c_h2;
    DevBuf<int32_t> i_off, i_len, i_msg, i_id;
    DevBuf<uint64_t> i_m1, i_m2;
    WireEnc* enc = nullptr;           // the encoder's outputs and scratch (wire_encode.cu)
};

static const int TB = 128;
static inline unsigned grid_for(int64_t n) { return (unsigned)ceil_div<int64_t>(n > 0 ? n : 1, TB); }

static int32_t wire_dict(Wire* w, Dict* d) {
    View* v = w->view;
    const int64_t tot = v->n + v->nj;
    if (w->table_epoch != v->epoch || w->T == 0) {
        uint32_t T = 1024;
        while ((int64_t)T < 2 * tot) T <<= 1;
        RAPID_CHECK(w->table.reserve(T));
        w->T = T;
        RAPID_CUDA(cudaStreamSynchronize(v->stream));
        RAPID_CUDA(cudaMemsetAsync(w->table.p, 0xff, (size_t)T * sizeof(int32_t), w->stream));
        if (tot) k_wire_table_build<<<grid_for(tot), TB, 0, w->stream>>>(tot, v->key.p, T, w->table.p);
        RAPID_KERNEL_CHECK();
        w->table_epoch = v->epoch;
    }
    d->T = w->T; d->table = w->table.p; d->key0 = v->key.p; d->hb = v->host_bytes.p; d->hoff = v->host_off.p; d->hport = v->port.p;
    return RAPID_OK;
}

static int32_t wire_read_scal(Wire* w) {
    RAPID_CUDA(cudaMemcpyAsync(w->h_sc.p, w->sc.p, sizeof(WireScal), cudaMemcpyDeviceToHost, w->stream));
    RAPID_CUDA(cudaStreamSynchronize(w->stream));
    return RAPID_OK;
}

// host: find the payload of field `field` (length-delimited) at the top level of [p, p+len); last occurrence wins
static bool host_find_field(const uint8_t* p, int64_t len, uint32_t field, const uint8_t** q, int64_t* ql) {
    Rd r{p, p + len, true};
    *q = nullptr; *ql = -1;
    while (r.ok && r.p < r.end) {
        const uint64_t tag = rd_varint(r);
        if (!r.ok) break;
        if ((tag >> 3) == 0) return false;
        if ((uint32_t)(tag >> 3) == field && (tag & 7) == 2) { if (!rd_len(r, q, ql)) return false; }
        else rd_skip(r, (uint32_t)(tag & 7));
    }
    return r.ok;
}

static const char* cons_name(int32_t kind) {
    switch (kind) {
        case RAPID_WIRE_FAST_ROUND_PHASE2B: return "FastRoundPhase2bMessage";
        case RAPID_WIRE_PHASE1A: return "Phase1aMessage";
        case RAPID_WIRE_PHASE1B: return "Phase1bMessage";
        case RAPID_WIRE_PHASE2A: return "Phase2aMessage";
        default: return "Phase2bMessage";
    }
}

// n serialized consensus messages of one kind -> the per-message fields and the flat list entries on the device.  Load-balanced:
// one thread per message walks the top level and counts list entries, a scan places them, one thread per message writes their
// byte ranges, one thread per ENTRY resolves it, one warp per message sums the fingerprint terms.  Whatever happens, the handle
// holds no consensus decode unless this returns RAPID_OK.
static int32_t wire_decode_consensus(Wire* w, int32_t kind, const uint8_t* bytes, const int64_t* off, int64_t n, uint32_t flags,
                                     int64_t* n_unknown_senders, int64_t* n_unknown_endpoints) {
    w->cons_kind = 0; w->cons_n = 0;
    if (n < 0 || (n && (!bytes || !off)) || n > 0x7ffffff0LL || kind < RAPID_WIRE_FAST_ROUND_PHASE2B || kind > RAPID_WIRE_PHASE2B) {
        set_error("bad arguments"); return RAPID_EINVAL;
    }
    if (n_unknown_senders) *n_unknown_senders = 0;
    if (n_unknown_endpoints) *n_unknown_endpoints = 0;
    if (n == 0) { w->cons_kind = kind; return RAPID_OK; }
    for (int64_t i = 0; i < n; ++i)
        if (off[i + 1] < off[i]) { set_error("off must be non-decreasing"); return RAPID_EINVAL; }
    // byte offsets inside the buffer are int32 (EpRef); every list entry takes at least 2 bytes, so their count fits int32 too
    if (off[0] < 0 || off[n] > 0x7ffffff0LL) { set_error("bad arguments: off must lie in [0, 0x7ffffff0]"); return RAPID_EINVAL; }
    const int64_t len = off[n] - off[0];
    DeviceGuard g(w->device);
    cudaStream_t s = w->stream;
    RAPID_CUDA(cudaEventRecord(w->ev0, s));
    Dict d;
    RAPID_CHECK(wire_dict(w, &d));
    RAPID_CHECK(w->buf.reserve((size_t)std::max<int64_t>(off[n], 1)));
    // keep the caller's offsets valid: copy [0, off[n]) (the prefix before off[0] is never read)
    if (len) RAPID_CUDA(cudaMemcpyAsync(w->buf.p + off[0], bytes + off[0], (size_t)len, cudaMemcpyHostToDevice, s));
    const size_t m = (size_t)n;
    RAPID_CHECK(w->c_off.reserve(m + 1)); RAPID_CHECK(w->c_cfg.reserve(m)); RAPID_CHECK(w->c_sender.reserve(m));
    RAPID_CHECK(w->c_ra_round.reserve(m)); RAPID_CHECK(w->c_ra_node.reserve(m)); RAPID_CHECK(w->c_rb_round.reserve(m));
    RAPID_CHECK(w->c_rb_node.reserve(m)); RAPID_CHECK(w->c_len.reserve(m)); RAPID_CHECK(w->c_pos.reserve(m));
    RAPID_CHECK(w->c_h1.reserve(m)); RAPID_CHECK(w->c_h2.reserve(m));
    RAPID_CUDA(cudaMemcpyAsync(w->c_off.p, off, (m + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    const int unwrap = (flags & RAPID_WIRE_REQUEST) ? 1 : 0;
    k_wire_begin<<<1, 1, 0, s>>>(w->sc.p);
    k_cons_top<<<grid_for(n), TB, 0, s>>>(n, w->buf.p, w->c_off.p, unwrap, kind, d, w->c_sender.p, w->c_cfg.p, w->c_ra_round.p,
                                          w->c_ra_node.p, w->c_rb_round.p, w->c_rb_node.p, w->c_len.p, w->sc.p);
    RAPID_KERNEL_CHECK();
    RAPID_CHECK(exclusive_scan_i32(w->c_pos.p, n, w->scan_sums, &w->sc.p->n_items, s, nullptr, w->c_len.p));
    RAPID_CHECK(wire_read_scal(w));
    const WireScal& sc = *w->h_sc.p;
    if (sc.bad_msg == INT_MAX) {
        const int64_t items = sc.n_items;
        if (items > 0) {
            const size_t k = (size_t)items;
            RAPID_CHECK(w->i_off.reserve(k)); RAPID_CHECK(w->i_len.reserve(k)); RAPID_CHECK(w->i_msg.reserve(k));
            RAPID_CHECK(w->i_id.reserve(k)); RAPID_CHECK(w->i_m1.reserve(k)); RAPID_CHECK(w->i_m2.reserve(k));
            k_cons_items<<<grid_for(n), TB, 0, s>>>(n, w->buf.p, w->c_off.p, unwrap, kind, w->c_len.p, w->c_pos.p, w->i_off.p, w->i_len.p,
                                                    w->i_msg.p);
            k_cons_resolve<<<grid_for(items), TB, 0, s>>>(items, w->buf.p, w->i_off.p, w->i_len.p, w->i_msg.p, d, w->i_id.p, w->i_m1.p,
                                                          w->i_m2.p, w->sc.p);
            RAPID_KERNEL_CHECK();
        }
        k_cons_reduce<<<(unsigned)ceil_div<int64_t>(n * 32, TB), TB, 0, s>>>(n, w->c_pos.p, w->c_len.p, w->i_m1.p, w->i_m2.p, w->c_h1.p,
                                                                             w->c_h2.p);
        RAPID_KERNEL_CHECK();
        RAPID_CUDA(cudaEventRecord(w->ev1, s));
        RAPID_CHECK(wire_read_scal(w));
        cudaEventElapsedTime(&w->last_ms, w->ev0, w->ev1);
    }
    if (sc.bad_msg != INT_MAX) { set_error("malformed %s at index %d", cons_name(kind), sc.bad_msg); return RAPID_EINVAL; }
    if (n_unknown_senders) *n_unknown_senders = sc.n_unknown_senders;
    if (n_unknown_endpoints) *n_unknown_endpoints = sc.n_unknown_endpoints;
    w->cons_kind = kind; w->cons_n = n;
    return RAPID_OK;
}

}  // namespace rapid

using namespace rapid;

struct rapid_wire : rapid::Wire {};

int32_t rapid::wire_consensus_dev(const rapid_wire* w, int32_t kind, WireMsgs* out) {
    if (!w) { set_error("NULL wire handle"); return RAPID_EINVAL; }
    if (w->cons_kind != kind) {
        set_error("the last decode on the wire handle is not a successful %s decode", cons_name(kind));
        return RAPID_EINVAL;
    }
    out->device = w->device; out->n = w->cons_n;
    out->sender = w->c_sender.p; out->cfg = w->c_cfg.p;
    out->rnd_round = w->c_ra_round.p; out->rnd_node = w->c_ra_node.p; out->vrnd_round = w->c_rb_round.p; out->vrnd_node = w->c_rb_node.p;
    out->h1 = w->c_h1.p; out->h2 = w->c_h2.p; out->len = w->c_len.p;
    return RAPID_OK;
}

void rapid::wire_enc_ctx(rapid_wire* w, WireEncCtx* out) {
    out->view = w->view; out->device = w->device; out->stream = w->stream; out->enc = &w->enc;
}

extern "C" {

int32_t rapid_wire_create(rapid_wire** out, rapid_view* v) {
    if (!out || !v) { set_error("NULL argument"); return RAPID_EINVAL; }
    *out = nullptr;
    DeviceGuard g(v->device);
    rapid_wire* w = new rapid_wire();
    w->view = v; w->device = v->device;
    int32_t rc = RAPID_OK;
    do {
        if (cudaStreamCreateWithFlags(&w->stream, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreate(&w->ev0) != cudaSuccess ||
            cudaEventCreate(&w->ev1) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "stream", __FILE__, __LINE__); break; }
        if ((rc = w->sc.reserve(1)) || (rc = w->h_sc.reserve(1))) break;
    } while (0);
    if (rc) { rapid_wire_destroy(w); return rc; }
    *out = w;
    return RAPID_OK;
}

int32_t rapid_wire_set_configuration(rapid_wire* w, int64_t cfg_id) {
    if (!w) { set_error("NULL handle"); return RAPID_EINVAL; }
    w->have_cfg = true; w->cur_cfg = cfg_id;
    return RAPID_OK;
}

int32_t rapid_wire_destroy(rapid_wire* w) {
    if (!w) return RAPID_OK;
    DeviceGuard g(w->device);
    if (w->stream) { cudaStreamSynchronize(w->stream); cudaStreamDestroy(w->stream); }
    if (w->ev0) cudaEventDestroy(w->ev0);
    if (w->ev1) cudaEventDestroy(w->ev1);
    wire_enc_free(w->enc);
    delete w;
    return RAPID_OK;
}

int32_t rapid_wire_decode_alerts(rapid_wire* w, const uint8_t* bytes, int64_t len, uint32_t flags, int64_t* n_messages, int64_t* n_cells,
                                 int64_t* n_dropped, int64_t* n_new_joiners, int32_t* sender_id) {
    if (w) w->cons_kind = 0;                                 // any decode replaces the last consensus decode
    if (!w || len < 0 || (len && !bytes) || len > 0x7ffffff0LL) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(w->device);
    cudaStream_t s = w->stream;
    w->M = 0; w->n_cells = 0;
    // ---- top level (host): BatchedAlertMessage { sender = 1; repeated AlertMessage messages = 3 }
    const uint8_t* body = bytes;
    int64_t blen = len;
    if (flags & RAPID_WIRE_REQUEST) {                        // RapidRequest.batchedAlertMessage = 3
        if (!host_find_field(bytes, len, 3, &body, &blen)) { set_error("malformed RapidRequest"); return RAPID_EINVAL; }
        if (blen < 0) { set_error("RapidRequest does not carry a BatchedAlertMessage"); return RAPID_EINVAL; }
    }
    std::vector<int64_t> moff;
    std::vector<int32_t> mlen;
    EpRef sender{0, 0, 0, 0};
    {
        Rd r{body, body + blen, true};
        bool ok = true;
        while (r.ok && r.p < r.end) {
            const uint64_t tag = rd_varint(r);
            if (!r.ok) break;
            const uint32_t f = (uint32_t)(tag >> 3), wt = (uint32_t)(tag & 7);
            const uint8_t* q; int64_t l;
            if (f == 3 && wt == 2) { if (rd_len(r, &q, &l)) { moff.push_back(q - bytes); mlen.push_back((int32_t)l); } }
            else if (f == 1 && wt == 2) { if (rd_len(r, &q, &l)) parse_endpoint(bytes, q, l, &sender, &ok); }
            else if (f == 0) r.ok = false;
            else rd_skip(r, wt);
        }
        if (!r.ok || !ok) { set_error("malformed BatchedAlertMessage"); return RAPID_EINVAL; }
    }
    const int64_t M = (int64_t)moff.size();
    RAPID_CUDA(cudaEventRecord(w->ev0, s));
    Dict d;
    RAPID_CHECK(wire_dict(w, &d));
    RAPID_CHECK(w->buf.reserve((size_t)std::max<int64_t>(len, 1)));
    if (len) RAPID_CUDA(cudaMemcpyAsync(w->buf.p, bytes, (size_t)len, cudaMemcpyHostToDevice, s));
    k_wire_begin<<<1, 1, 0, s>>>(w->sc.p);
    if (sender.present) k_wire_sender<<<1, 1, 0, s>>>(w->buf.p, sender, d, w->sc.p);
    RAPID_KERNEL_CHECK();
    int64_t new_joiners = 0;
    if (M > 0) {
        RAPID_CHECK(w->moff.reserve((size_t)M)); RAPID_CHECK(w->mlen.reserve((size_t)M)); RAPID_CHECK(w->need.reserve((size_t)M));
        RAPID_CHECK(w->cnt.reserve((size_t)M)); RAPID_CHECK(w->pos.reserve((size_t)M)); RAPID_CHECK(w->rec.reserve((size_t)M));
        RAPID_CUDA(cudaMemcpyAsync(w->moff.p, moff.data(), (size_t)M * sizeof(int64_t), cudaMemcpyHostToDevice, s));
        RAPID_CUDA(cudaMemcpyAsync(w->mlen.p, mlen.data(), (size_t)M * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        k_wire_parse_alerts<<<grid_for(M), TB, 0, s>>>(M, w->buf.p, w->moff.p, w->mlen.p, d, w->rec.p, w->need.p, w->sc.p, w->have_cfg ? 1 : 0, w->cur_cfg);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(wire_read_scal(w));
        if (w->h_sc.p->bad_msg != INT_MAX) { set_error("malformed AlertMessage at index %d", w->h_sc.p->bad_msg); return RAPID_EINVAL; }
        if (w->h_sc.p->n_need > 0) {
            // joiners announced by UP alerts: register them in order of first appearance, then resolve again
            std::vector<int32_t> need((size_t)M);
            std::vector<MsgRec> rec((size_t)M);
            RAPID_CUDA(cudaMemcpyAsync(need.data(), w->need.p, (size_t)M * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
            RAPID_CUDA(cudaMemcpyAsync(rec.data(), w->rec.p, (size_t)M * sizeof(MsgRec), cudaMemcpyDeviceToHost, s));
            RAPID_CUDA(cudaStreamSynchronize(s));
            std::map<std::pair<std::string, int32_t>, int> seen;
            std::vector<uint8_t> hb;
            std::vector<int32_t> off(1, 0), port;
            for (int64_t m = 0; m < M; ++m) {
                if (!need[(size_t)m]) continue;
                const EpRef& e = rec[(size_t)m].dst;
                std::pair<std::string, int32_t> k(std::string((const char*)bytes + e.off, (size_t)e.len), e.port);
                if (seen.count(k)) continue;
                seen[k] = 1;
                hb.insert(hb.end(), bytes + e.off, bytes + e.off + e.len);
                off.push_back(off.back() + e.len);
                port.push_back(e.port);
            }
            new_joiners = (int64_t)port.size();
            static const uint8_t dummy = 0;
            int32_t first = 0;
            RAPID_CHECK(rapid_view_register_joiners(w->view, new_joiners, hb.empty() ? &dummy : hb.data(), off.data(), port.data(), &first));
            RAPID_CHECK(wire_dict(w, &d));
            k_wire_relookup<<<grid_for(M), TB, 0, s>>>(M, w->buf.p, d, w->rec.p);
            if (sender.present) k_wire_sender<<<1, 1, 0, s>>>(w->buf.p, sender, d, w->sc.p);
            RAPID_KERNEL_CHECK();
        }
        k_wire_counts<<<grid_for(M), TB, 0, s>>>(M, w->rec.p, w->cnt.p, w->sc.p);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(exclusive_scan_i32_to(w->cnt.p, w->pos.p, M, w->scan_sums, s));
        // every ring number is at least one byte on the wire: len bounds the number of cells
        const size_t cap = (size_t)std::max<int64_t>(len, 1);
        RAPID_CHECK(w->o_src.reserve(cap)); RAPID_CHECK(w->o_dst.reserve(cap)); RAPID_CHECK(w->o_ring.reserve(cap));
        RAPID_CHECK(w->o_status.reserve(cap)); RAPID_CHECK(w->o_cfg.reserve(cap));
        k_wire_emit<<<grid_for(M), TB, 0, s>>>(M, w->buf.p, w->moff.p, w->mlen.p, w->rec.p, w->cnt.p, w->pos.p, w->o_src.p, w->o_dst.p,
                                               w->o_ring.p, w->o_status.p, w->o_cfg.p, w->sc.p);
        RAPID_KERNEL_CHECK();
    }
    RAPID_CUDA(cudaEventRecord(w->ev1, s));
    RAPID_CHECK(wire_read_scal(w));
    cudaEventElapsedTime(&w->last_ms, w->ev0, w->ev1);
    w->M = M; w->n_cells = w->h_sc.p->n_cells;
    if (n_messages) *n_messages = M;
    if (n_cells) *n_cells = w->n_cells;
    if (n_dropped) *n_dropped = w->h_sc.p->n_dropped;
    if (n_new_joiners) *n_new_joiners = new_joiners;
    if (sender_id) *sender_id = w->h_sc.p->sender_id;
    return RAPID_OK;
}

int32_t rapid_wire_cells_dev(const rapid_wire* w, const int32_t** src, const int32_t** dst, const uint8_t** ring, const uint8_t** status,
                             const int64_t** cfg) {
    if (!w) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (src) *src = w->o_src.p;
    if (dst) *dst = w->o_dst.p;
    if (ring) *ring = w->o_ring.p;
    if (status) *status = w->o_status.p;
    if (cfg) *cfg = w->o_cfg.p;
    return RAPID_OK;
}

int32_t rapid_wire_read_cells(const rapid_wire* w, int32_t* src, int32_t* dst, uint8_t* ring, uint8_t* status, int64_t* cfg) {
    if (!w) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(w->device);
    const size_t n = (size_t)w->n_cells;
    if (n == 0) return RAPID_OK;
    cudaStream_t s = w->stream;
    if (src) RAPID_CUDA(cudaMemcpyAsync(src, w->o_src.p, n * 4, cudaMemcpyDeviceToHost, s));
    if (dst) RAPID_CUDA(cudaMemcpyAsync(dst, w->o_dst.p, n * 4, cudaMemcpyDeviceToHost, s));
    if (ring) RAPID_CUDA(cudaMemcpyAsync(ring, w->o_ring.p, n, cudaMemcpyDeviceToHost, s));
    if (status) RAPID_CUDA(cudaMemcpyAsync(status, w->o_status.p, n, cudaMemcpyDeviceToHost, s));
    if (cfg) RAPID_CUDA(cudaMemcpyAsync(cfg, w->o_cfg.p, n * 8, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

int32_t rapid_wire_read_messages(const rapid_wire* cw, int32_t* dst, uint8_t* status, int32_t* n_rings, int64_t* node_high, int64_t* node_low,
                                 uint8_t* has_node_id, int64_t* meta_off, int32_t* meta_len) {
    rapid_wire* w = const_cast<rapid_wire*>(cw);             // uses the handle's staging buffers; logically const
    if (!w) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(w->device);
    const int64_t M = w->M;
    if (M == 0) return RAPID_OK;
    cudaStream_t s = w->stream;
    const size_t m = (size_t)M;
    RAPID_CHECK(w->t_i32a.reserve(m)); RAPID_CHECK(w->t_i32b.reserve(m)); RAPID_CHECK(w->t_i32c.reserve(m));
    RAPID_CHECK(w->t_i64a.reserve(m)); RAPID_CHECK(w->t_i64b.reserve(m)); RAPID_CHECK(w->t_i64c.reserve(m));
    RAPID_CHECK(w->t_u8a.reserve(m)); RAPID_CHECK(w->t_u8b.reserve(m));
    k_wire_msg_fields<<<grid_for(M), TB, 0, s>>>(M, w->rec.p, w->t_i32a.p, w->t_u8a.p, w->t_i32b.p, w->t_i64a.p, w->t_i64b.p, w->t_u8b.p,
                                                 w->t_i64c.p, w->t_i32c.p);
    RAPID_KERNEL_CHECK();
    if (dst) RAPID_CUDA(cudaMemcpyAsync(dst, w->t_i32a.p, m * 4, cudaMemcpyDeviceToHost, s));
    if (status) RAPID_CUDA(cudaMemcpyAsync(status, w->t_u8a.p, m, cudaMemcpyDeviceToHost, s));
    if (n_rings) RAPID_CUDA(cudaMemcpyAsync(n_rings, w->t_i32b.p, m * 4, cudaMemcpyDeviceToHost, s));
    if (node_high) RAPID_CUDA(cudaMemcpyAsync(node_high, w->t_i64a.p, m * 8, cudaMemcpyDeviceToHost, s));
    if (node_low) RAPID_CUDA(cudaMemcpyAsync(node_low, w->t_i64b.p, m * 8, cudaMemcpyDeviceToHost, s));
    if (has_node_id) RAPID_CUDA(cudaMemcpyAsync(has_node_id, w->t_u8b.p, m, cudaMemcpyDeviceToHost, s));
    if (meta_off) RAPID_CUDA(cudaMemcpyAsync(meta_off, w->t_i64c.p, m * 8, cudaMemcpyDeviceToHost, s));
    if (meta_len) RAPID_CUDA(cudaMemcpyAsync(meta_len, w->t_i32c.p, m * 4, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

int32_t rapid_wire_decode_votes(rapid_wire* w, const uint8_t* bytes, const int64_t* off, int64_t n, uint32_t flags, int32_t* sender,
                                int64_t* vote_cfg, uint64_t* proposal_hash, uint64_t* proposal_hash2, int32_t* proposal_len) {
    if (!w) { set_error("bad arguments"); return RAPID_EINVAL; }
    RAPID_CHECK(wire_decode_consensus(w, RAPID_WIRE_FAST_ROUND_PHASE2B, bytes, off, n, flags, nullptr, nullptr));
    // (a vote naming an endpoint outside the dictionary is NOT an error: see ep_fp_terms)
    if (n == 0) return RAPID_OK;
    DeviceGuard g(w->device);
    cudaStream_t s = w->stream;
    const size_t m = (size_t)n;
    if (sender) RAPID_CUDA(cudaMemcpyAsync(sender, w->c_sender.p, m * 4, cudaMemcpyDeviceToHost, s));
    if (vote_cfg) RAPID_CUDA(cudaMemcpyAsync(vote_cfg, w->c_cfg.p, m * 8, cudaMemcpyDeviceToHost, s));
    if (proposal_hash) RAPID_CUDA(cudaMemcpyAsync(proposal_hash, w->c_h1.p, m * 8, cudaMemcpyDeviceToHost, s));
    if (proposal_hash2) RAPID_CUDA(cudaMemcpyAsync(proposal_hash2, w->c_h2.p, m * 8, cudaMemcpyDeviceToHost, s));
    if (proposal_len) RAPID_CUDA(cudaMemcpyAsync(proposal_len, w->c_len.p, m * 4, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

int32_t rapid_wire_decode_consensus(rapid_wire* w, int32_t kind, const uint8_t* bytes, const int64_t* off, int64_t n, uint32_t flags,
                                    int64_t* n_unknown_senders, int64_t* n_unknown_endpoints) {
    if (!w) { set_error("NULL handle"); return RAPID_EINVAL; }
    return wire_decode_consensus(w, kind, bytes, off, n, flags, n_unknown_senders, n_unknown_endpoints);
}

int32_t rapid_wire_read_consensus(const rapid_wire* w, int32_t* sender, int64_t* cfg, int32_t* rnd_round, int32_t* rnd_node,
                                  int32_t* vrnd_round, int32_t* vrnd_node, uint64_t* h1, uint64_t* h2, int32_t* len) {
    if (!w) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (!w->cons_kind) { set_error("no consensus decode on this handle"); return RAPID_EINVAL; }
    const size_t m = (size_t)w->cons_n;
    if (m == 0) return RAPID_OK;
    DeviceGuard g(w->device);
    cudaStream_t s = w->stream;
    if (sender) RAPID_CUDA(cudaMemcpyAsync(sender, w->c_sender.p, m * 4, cudaMemcpyDeviceToHost, s));
    if (cfg) RAPID_CUDA(cudaMemcpyAsync(cfg, w->c_cfg.p, m * 8, cudaMemcpyDeviceToHost, s));
    if (rnd_round) RAPID_CUDA(cudaMemcpyAsync(rnd_round, w->c_ra_round.p, m * 4, cudaMemcpyDeviceToHost, s));
    if (rnd_node) RAPID_CUDA(cudaMemcpyAsync(rnd_node, w->c_ra_node.p, m * 4, cudaMemcpyDeviceToHost, s));
    if (vrnd_round) RAPID_CUDA(cudaMemcpyAsync(vrnd_round, w->c_rb_round.p, m * 4, cudaMemcpyDeviceToHost, s));
    if (vrnd_node) RAPID_CUDA(cudaMemcpyAsync(vrnd_node, w->c_rb_node.p, m * 4, cudaMemcpyDeviceToHost, s));
    if (h1) RAPID_CUDA(cudaMemcpyAsync(h1, w->c_h1.p, m * 8, cudaMemcpyDeviceToHost, s));
    if (h2) RAPID_CUDA(cudaMemcpyAsync(h2, w->c_h2.p, m * 8, cudaMemcpyDeviceToHost, s));
    if (len) RAPID_CUDA(cudaMemcpyAsync(len, w->c_len.p, m * 4, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

int32_t rapid_wire_consensus_value(const rapid_wire* w, int64_t index, int32_t* out_ids, int32_t cap, int32_t* out_len) {
    if (!w) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (!w->cons_kind) { set_error("no consensus decode on this handle"); return RAPID_EINVAL; }
    if (index < 0 || index >= w->cons_n || cap < 0 || (cap > 0 && !out_ids)) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(w->device);
    cudaStream_t s = w->stream;
    int32_t at = 0, len = 0;
    RAPID_CUDA(cudaMemcpyAsync(&at, w->c_pos.p + index, 4, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaMemcpyAsync(&len, w->c_len.p + index, 4, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    const int32_t k = std::min(cap, len);
    if (k > 0) {
        RAPID_CUDA(cudaMemcpyAsync(out_ids, w->i_id.p + at, (size_t)k * 4, cudaMemcpyDeviceToHost, s));
        RAPID_CUDA(cudaStreamSynchronize(s));
    }
    if (out_len) *out_len = len;
    return RAPID_OK;
}

int32_t rapid_wire_last_device_ms(const rapid_wire* w, float* total_ms) {
    if (!w || !total_ms) return RAPID_EINVAL;
    *total_ms = w->last_ms;
    return RAPID_OK;
}

}  // extern "C"
