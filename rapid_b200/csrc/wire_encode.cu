// Wire-format egress (DESIGN §4.14): the messages a virtual cluster sends, serialized on the device as the protobuf runtime
// serializes them (rapid.proto:13-17, 95-129), optionally wrapped in RapidRequest.
//
// A message is a HEADER plus, for the kinds whose last field is a list, a BODY shared by every message that carries the same
// list: canonical bytes = header ++ body, because fields are serialized in field-number order and the list is the highest.
// Bodies are the distinct (h1, h2, len) fingerprints of the lists (the identity the tally already counts votes by), grouped on the
// device by the proposal census's grouping (group_proposals, cd_census.cu); each is encoded once, one thread per list ENTRY, from
// the canonical list of its lowest sender.  Every kind is count -> exclusive scan -> emit, the scheme of the decoder (wire.cu),
// with the int32 scans of scan.cuh.
// Outputs are double-buffered: an encode writes the spare set and swaps on success, so a refused or failed encode leaves the
// previous outputs as they were.
#include <limits.h>

#include <algorithm>
#include <map>
#include <tuple>
#include <vector>

#include "cd_internal.cuh"
#include "common.cuh"
#include "scan.cuh"
#include "wire_internal.cuh"

namespace rapid {

// ------------------------------------------------------------------ protobuf primitives
RAPID_HD int32_t vsz(uint64_t v) {                  // bytes of a varint
    int32_t n = 1;
    while (v >= 0x80) { v >>= 7; ++n; }
    return n;
}
// an int32 / int64 / enum field is the varint of the value sign-extended to 64 bits: a negative one takes 10 bytes
RAPID_HD uint64_t sx(int64_t v) { return (uint64_t)v; }
RAPID_HD int32_t msg_field(int32_t content) { return 1 + vsz((uint64_t)content) + content; }   // tag (field <= 15), length, content

__device__ __forceinline__ uint8_t* put_varint(uint8_t* p, uint64_t v) {
    while (v >= 0x80) { *p++ = (uint8_t)(v | 0x80); v >>= 7; }
    *p++ = (uint8_t)v;
    return p;
}

// the view's endpoint table (members, then registered joiners)
struct EpTab {
    const uint8_t* hb;
    const int32_t* hoff;
    const int32_t* port;
};
// Endpoint content: hostname (1, omitted when empty), port (2, omitted when 0)
__device__ __forceinline__ int32_t ep_size(const EpTab& t, int32_t id) {
    const int32_t hl = t.hoff[id + 1] - t.hoff[id], port = t.port[id];
    return (hl ? 1 + vsz((uint64_t)hl) + hl : 0) + (port ? 1 + vsz(sx(port)) : 0);
}
// a SET Endpoint field: serialized even when its content is empty
__device__ uint8_t* put_ep_field(uint8_t* p, uint8_t tag, const EpTab& t, int32_t id) {
    const int32_t hl = t.hoff[id + 1] - t.hoff[id], port = t.port[id];
    *p++ = tag;
    p = put_varint(p, (uint64_t)ep_size(t, id));
    if (hl) {
        *p++ = 0x0A;
        p = put_varint(p, (uint64_t)hl);
        const uint8_t* s = t.hb + t.hoff[id];
        for (int32_t i = 0; i < hl; ++i) p[i] = s[i];
        p += hl;
    }
    if (port) { *p++ = 0x10; p = put_varint(p, sx(port)); }
    return p;
}

struct EncScal {
    int32_t n_msgs, n_bodies, n_heads, n_entries;
    int32_t hdr_bytes, body_bytes, alert_bytes, pad_;
    unsigned long long bytes64;        // the entries' bytes summed in 64 bits: an encode whose offsets would not fit int32 is refused
};

// ------------------------------------------------------------------ alert batches (rapid.proto:95-110)
struct AlertIn {
    int32_t n;
    const int32_t* obs;
    const int32_t* subj;
    const uint16_t* mask;
    const uint8_t* status;             // per cell
    const int64_t* cfg;                // per cell
    const int32_t* cpos;               // first cell of each alert
    const int64_t* nid_hi;             // NodeIds by view id, NULL: the view holds none (zero halves)
    const int64_t* nid_lo;
};

__device__ __forceinline__ int32_t nid_size(int64_t hi, int64_t lo) { return (hi ? 1 + vsz(sx(hi)) : 0) + (lo ? 1 + vsz(sx(lo)) : 0); }

struct AlertFields {
    uint8_t st;
    int64_t cfg, hi, lo;
};
// AlertMessage content as MembershipService builds it: edgeSrc, edgeDst, edgeStatus (omitted when UP), configurationId (omitted
// when 0), ringNumber packed and ascending; an UP alert also sets nodeId (:250) and metadata (:252, empty: the device holds none)
__device__ int32_t alert_size(const AlertIn& a, const EpTab& t, int32_t i, AlertFields* f) {
    const int32_t c = a.cpos[i];
    f->st = a.status[c];
    f->cfg = a.cfg[c];
    f->hi = f->lo = 0;
    const int32_t nr = __popc((uint32_t)a.mask[i]);
    int32_t s = msg_field(ep_size(t, a.obs[i])) + msg_field(ep_size(t, a.subj[i])) + (f->st ? 2 : 0) +
                (f->cfg ? 1 + vsz(sx(f->cfg)) : 0) + 1 + vsz((uint64_t)nr) + nr;   // ring numbers < RAPID_MAX_K: one byte each
    if (f->st == RAPID_EDGE_UP) {
        if (a.nid_hi) { f->hi = a.nid_hi[a.subj[i]]; f->lo = a.nid_lo[a.subj[i]]; }
        s += msg_field(nid_size(f->hi, f->lo)) + 2;
    }
    return s;
}

__global__ void k_enc_popc(int32_t n, const uint16_t* __restrict__ mask, int32_t* __restrict__ cnt) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) cnt[i] = __popc((uint32_t)mask[i]);
}
// per alert: the size of its entry in BatchedAlertMessage.messages, and whether it opens a sender's batch
__global__ void k_enc_alert_sizes(AlertIn a, EpTab t, int32_t* __restrict__ esz, int32_t* __restrict__ head, EncScal* __restrict__ sc) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    AlertFields f;
    const int32_t e = msg_field(alert_size(a, t, i, &f));
    esz[i] = e;
    head[i] = (i == 0 || a.obs[i] != a.obs[i - 1]) ? 1 : 0;
    atomicAdd(&sc->bytes64, (unsigned long long)e);
}
// per batch (the thread of the alert that opens it): its first alert, its header size and the whole message's size
__global__ void k_enc_batch_sizes(int32_t n, const int32_t* __restrict__ obs, const int32_t* __restrict__ head,
                                  const int32_t* __restrict__ bpos, const int32_t* __restrict__ epos, const EncScal* __restrict__ sc,
                                  EpTab t, int wrap, int32_t* __restrict__ start, int32_t* __restrict__ hlen, int32_t* __restrict__ msz) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !head[i]) return;
    const int32_t b = bpos[i];
    int32_t j = i + 1;                                                       // the next batch's first alert: a batch is <= ~2K alerts
    while (j < n && !head[j]) ++j;
    const int32_t body = (j < n ? epos[j] : sc->alert_bytes) - epos[i];
    const int32_t content = msg_field(ep_size(t, obs[i])) + body;
    const int32_t h = (wrap ? 1 + vsz((uint64_t)content) : 0) + content - body;
    start[b] = i; hlen[b] = h; msz[b] = h + body;
}
// the batch's header: [RapidRequest tag 3, length] BatchedAlertMessage.sender
__global__ void k_enc_batch_emit(int32_t nb, const int32_t* __restrict__ start, const int32_t* __restrict__ hlen,
                                 const int32_t* __restrict__ msz, const int32_t* __restrict__ hpos, const int32_t* __restrict__ obs,
                                 EpTab t, int wrap, int32_t* __restrict__ m_snd, uint8_t* __restrict__ out) {
    const int32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    uint8_t* p = out + hpos[b];
    const int32_t s = obs[start[b]];
    m_snd[b] = s;
    if (wrap) {
        const int32_t content = msz[b] - hlen[b] + msg_field(ep_size(t, s));
        *p++ = 0x1A;
        p = put_varint(p, (uint64_t)content);
    }
    put_ep_field(p, 0x0A, t, s);
}
// per alert: its entry (tag 3, length, AlertMessage) at its place in its sender's message
__global__ void k_enc_alert_emit(AlertIn a, EpTab t, const int32_t* __restrict__ head, const int32_t* __restrict__ bpos,
                                 const int32_t* __restrict__ epos, const int32_t* __restrict__ start, const int32_t* __restrict__ hlen,
                                 const int32_t* __restrict__ hpos, uint8_t* __restrict__ out) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    const int32_t b = bpos[i] + head[i] - 1;                                 // bpos: exclusive count of batch openers
    uint8_t* p = out + hpos[b] + hlen[b] + (epos[i] - epos[start[b]]);
    AlertFields f;
    const int32_t sz = alert_size(a, t, i, &f);
    *p++ = 0x1A;
    p = put_varint(p, (uint64_t)sz);
    p = put_ep_field(p, 0x0A, t, a.obs[i]);
    p = put_ep_field(p, 0x12, t, a.subj[i]);
    if (f.st) { *p++ = 0x18; *p++ = f.st; }
    if (f.cfg) { *p++ = 0x20; p = put_varint(p, sx(f.cfg)); }
    const uint32_t m = a.mask[i];
    *p++ = 0x2A;
    *p++ = (uint8_t)__popc(m);
    for (uint32_t r = 0; r < 16; ++r) if ((m >> r) & 1u) *p++ = (uint8_t)r;
    if (f.st == RAPID_EDGE_UP) {
        *p++ = 0x32;
        p = put_varint(p, (uint64_t)nid_size(f.hi, f.lo));
        if (f.hi) { *p++ = 0x08; p = put_varint(p, sx(f.hi)); }
        if (f.lo) { *p++ = 0x10; p = put_varint(p, sx(f.lo)); }
        *p++ = 0x3A; *p++ = 0x00;
    }
}

// ------------------------------------------------------------------ list-carrying messages (rapid.proto:124-169)
// One slot per candidate message: a detector receiver (FastRoundPhase2bMessage: it sends iff it announced in the last call) or a
// pending acceptor answer (Phase1bMessage, Phase2bMessage: every slot sends).  Each kind ends with its endpoint list.
struct ListIn {
    int32_t n;
    int32_t kind;                       // RAPID_WIRE_FAST_ROUND_PHASE2B, RAPID_WIRE_PHASE1B or RAPID_WIRE_PHASE2B
    int wrap;
    int64_t cfg;
    const uint32_t* rflags;             // votes; NULL: every slot sends
    const int32_t* acc;                 // answers: the sender's acceptor index, a ring-0 position; NULL: rbegin + slot
    int64_t rbegin;
    const int32_t* ring0;
    const int64_t* vrnd;                // Phase1b: per slot
    int64_t rank;                       // Phase1b / Phase2b: rnd (packed, see pack_rank)
};
__device__ __forceinline__ bool list_sends(const ListIn& L, int32_t s) { return !L.rflags || (L.rflags[s] & RF_ANN_NOW); }
__device__ __forceinline__ int32_t list_sender(const ListIn& L, int32_t s) { return L.ring0[L.acc ? L.acc[s] : L.rbegin + s]; }
// Rank {round = 1, nodeIndex = 2}, int32 fields
__device__ __forceinline__ int32_t rank_size(int64_t p) {
    const int32_t r = rank_round(p), q = rank_node(p);
    return (r ? 1 + vsz(sx(r)) : 0) + (q ? 1 + vsz(sx(q)) : 0);
}
__device__ uint8_t* put_rank_field(uint8_t* p, uint8_t tag, int64_t rk) {        // a SET Rank: written even when (0, 0)
    const int32_t r = rank_round(rk), q = rank_node(rk);
    *p++ = tag;
    p = put_varint(p, (uint64_t)rank_size(rk));
    if (r) { *p++ = 0x08; p = put_varint(p, sx(r)); }
    if (q) { *p++ = 0x10; p = put_varint(p, sx(q)); }
    return p;
}
RAPID_HD uint8_t list_tag(int32_t kind) {                                  // endpoints = 3 / vval = 5 / endpoints = 4
    return kind == RAPID_WIRE_FAST_ROUND_PHASE2B ? 0x1A : kind == RAPID_WIRE_PHASE1B ? 0x2A : 0x22;
}

__global__ void k_enc_send(ListIn L, int32_t* __restrict__ send) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < L.n) send[s] = list_sends(L, s) ? 1 : 0;
}
// one thread per list entry: its size as a repeated Endpoint field
__global__ void k_enc_entry_sizes(int32_t n, const int32_t* __restrict__ ids, EpTab t, int32_t* __restrict__ sz, EncScal* __restrict__ sc) {
    const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int32_t s = msg_field(ep_size(t, ids[j]));
    sz[j] = s;
    atomicAdd(&sc->bytes64, (unsigned long long)s);
}
__global__ void k_enc_entry_emit(int32_t n, const int32_t* __restrict__ ids, EpTab t, uint8_t tag, const int32_t* __restrict__ pos,
                                 uint8_t* __restrict__ out) {
    const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) put_ep_field(out + pos[j], tag, t, ids[j]);
}
// body b = entries [first[b], first[b] + len[b]), len[b] > 0: its byte range
__global__ void k_enc_body_off(int32_t nb, const int32_t* __restrict__ first, const int32_t* __restrict__ pos,
                               const EncScal* __restrict__ sc, int64_t* __restrict__ boff) {
    const int32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b > nb) return;
    boff[b] = b < nb ? pos[first[b]] : sc->body_bytes;
}
// per sending slot: header = [RapidRequest tag, length] sender, configurationId (omitted when 0), and the kind's ranks (Phase1b:
// rnd, vrnd; Phase2b: rnd; both set, so written even when (0, 0))
__device__ __forceinline__ int32_t list_header(const ListIn& L, const EpTab& t, const int32_t* bid, const int64_t* boff, int32_t s,
                                               int32_t* content) {
    const int32_t b = bid[s];
    const int32_t body = b >= 0 ? (int32_t)(boff[b + 1] - boff[b]) : 0;
    int32_t own = msg_field(ep_size(t, list_sender(L, s))) + (L.cfg ? 1 + vsz(sx(L.cfg)) : 0);
    if (L.kind != RAPID_WIRE_FAST_ROUND_PHASE2B) own += msg_field(rank_size(L.rank));
    if (L.kind == RAPID_WIRE_PHASE1B) own += msg_field(rank_size(L.vrnd[s]));
    *content = own + body;
    return (L.wrap ? 1 + vsz((uint64_t)*content) : 0) + own;
}
__global__ void k_enc_list_sizes(ListIn L, EpTab t, const int32_t* __restrict__ send, const int32_t* __restrict__ mpos,
                                 const int32_t* __restrict__ bid, const int64_t* __restrict__ boff, int32_t* __restrict__ hsz) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= L.n || !send[s]) return;
    int32_t content;
    hsz[mpos[s]] = list_header(L, t, bid, boff, s, &content);
}
__global__ void k_enc_list_emit(ListIn L, EpTab t, const int32_t* __restrict__ send, const int32_t* __restrict__ mpos,
                                const int32_t* __restrict__ bid, const int64_t* __restrict__ boff, const int32_t* __restrict__ hpos,
                                int32_t* __restrict__ m_bid, int32_t* __restrict__ m_snd, uint8_t* __restrict__ out) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= L.n || !send[s]) return;
    const int32_t m = mpos[s];
    int32_t content;
    list_header(L, t, bid, boff, s, &content);
    uint8_t* p = out + hpos[m];
    if (L.wrap) { *p++ = (uint8_t)((L.kind << 3) | 2); p = put_varint(p, (uint64_t)content); }
    const int32_t snd = list_sender(L, s);
    p = put_ep_field(p, 0x0A, t, snd);
    if (L.cfg) { *p++ = 0x10; p = put_varint(p, sx(L.cfg)); }
    if (L.kind != RAPID_WIRE_FAST_ROUND_PHASE2B) p = put_rank_field(p, 0x1A, L.rank);
    if (L.kind == RAPID_WIRE_PHASE1B) p = put_rank_field(p, 0x22, L.vrnd[s]);
    m_bid[m] = bid[s];
    m_snd[m] = snd;
}

// ------------------------------------------------------------------ offsets, sizes
__global__ void k_enc_off64(int32_t n, const int32_t* __restrict__ pos, const int32_t* __restrict__ total, int64_t* __restrict__ off) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) off[i] = pos[i];
    if (i == n) off[i] = *total;
}
__global__ void k_enc_fill(int32_t n, int32_t v, int32_t* __restrict__ a) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] = v;
}
__global__ void k_enc_sizes(int64_t n, const int64_t* __restrict__ hoff, const int32_t* __restrict__ bid, const int64_t* __restrict__ boff,
                            int64_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t b = bid[i];
    out[i] = hoff[i + 1] - hoff[i] + (b >= 0 ? boff[b + 1] - boff[b] : 0);
}

// ------------------------------------------------------------------ state
struct EncOut {
    int64_t n = 0, n_bodies = 0, hdr_bytes = 0, body_bytes = 0;
    DevBuf<uint8_t> hdr, bodies;
    DevBuf<int64_t> hoff, boff;        // [n + 1], [n_bodies + 1]
    DevBuf<int32_t> bid;               // [n]: body of each message, -1 for none
    DevBuf<int32_t> snd;               // [n]: view id of each message's sender
};

struct WireEnc {
    EncOut out[2];
    int cur = 0;                       // out[cur] holds the last successful encode
    DevBuf<int32_t> a, b, c, d, e, f, g, scan_sums;
    DevBuf<int32_t> ids, epos;
    DevBuf<int64_t> sizes;
    ProposalGroups grp;                // the bodies of list-carrying messages (group_bodies), never a detector's census
    DevBuf<int32_t> cls;               // [n]: body of every slot, -1 for none
    DevBuf<EncScal> sc;
    PinnedBuf<EncScal> h_sc;
    // the lists already fetched as ids, by (h1, h2, len), for the view's member_epoch `lists_epoch`: a vval or Phase2a value is
    // looked up here first (the votes encoded earlier hold every proposal the acceptors can have registered)
    std::map<std::tuple<uint64_t, uint64_t, int32_t>, std::vector<int32_t>> lists;
    uint64_t lists_epoch = 0;
};

static const int TB = 256;
static inline unsigned grid_for(int64_t n) { return (unsigned)ceil_div<int64_t>(n > 0 ? n : 1, TB); }

void wire_enc_free(WireEnc* e) { delete e; }

static int32_t enc_get(rapid_wire* w, WireEncCtx* ctx, WireEnc** out) {
    wire_enc_ctx(w, ctx);
    if (!*ctx->enc) {
        WireEnc* e = new WireEnc();
        int32_t rc;
        if ((rc = e->sc.reserve(1)) || (rc = e->h_sc.reserve(1))) { delete e; return rc; }
        for (EncOut& o : e->out) {                                   // an empty encode: offsets {0}
            if ((rc = o.hoff.reserve(1)) || (rc = o.boff.reserve(1))) { delete e; return rc; }
            RAPID_CUDA(cudaMemsetAsync(o.hoff.p, 0, sizeof(int64_t), ctx->stream));
            RAPID_CUDA(cudaMemsetAsync(o.boff.p, 0, sizeof(int64_t), ctx->stream));
        }
        *ctx->enc = e;
    }
    *out = *ctx->enc;
    return RAPID_OK;
}

static int32_t enc_read_scal(WireEnc* e, cudaStream_t s) {
    RAPID_CUDA(cudaMemcpyAsync(e->h_sc.p, e->sc.p, sizeof(EncScal), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

static EpTab ep_tab(const View* v) { return EpTab{v->host_bytes.p, v->host_off.p, v->port.p}; }

static const int64_t ENC_LIMIT = 0x7ff00000LL;   // bytes of one encode's headers or bodies (int32 offsets in the scans)

static int32_t too_big() { set_error("the encoded messages would exceed 2^31 bytes"); return RAPID_ENOMEM; }

// BatchedAlertMessage of every sender of the fdet's last interval
static int32_t encode_alerts(WireEnc* e, const WireEncCtx& ctx, const FdetInterval& in, uint32_t flags) {
    cudaStream_t s = ctx.stream;
    EncOut& o = e->out[1 - e->cur];
    const int32_t n = (int32_t)in.n_alerts;
    const int wrap = (flags & RAPID_WIRE_REQUEST) ? 1 : 0;
    const EpTab t = ep_tab(ctx.view);
    RAPID_CUDA(cudaMemsetAsync(e->sc.p, 0, sizeof(EncScal), s));
    int64_t nb = 0, hbytes = 0;
    if (n > 0) {
        const size_t N = (size_t)n;
        RAPID_CHECK(e->a.reserve(N)); RAPID_CHECK(e->b.reserve(N)); RAPID_CHECK(e->c.reserve(N)); RAPID_CHECK(e->d.reserve(N));
        RAPID_CHECK(e->f.reserve(N)); RAPID_CHECK(e->g.reserve(N)); RAPID_CHECK(e->e.reserve(N + 1));
        int32_t *cpos = e->a.p, *esz = e->b.p, *epos = e->b.p, *head = e->c.p, *bpos = e->d.p;
        int32_t *start = e->e.p, *hlen = e->f.p, *msz = e->g.p;
        k_enc_popc<<<grid_for(n), TB, 0, s>>>(n, in.mask, cpos);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(exclusive_scan_i32(cpos, n, e->scan_sums, nullptr, s, nullptr));
        const bool nid = ctx.view->has_node_ids;
        const AlertIn a{n, in.obs, in.subj, in.mask, in.cell_status, in.cell_cfg, cpos, nid ? ctx.view->node_hi.p : nullptr,
                        nid ? ctx.view->node_lo.p : nullptr};
        k_enc_alert_sizes<<<grid_for(n), TB, 0, s>>>(a, t, esz, head, e->sc.p);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(enc_read_scal(e, s));
        // + one sender field per alert at most: a bound on the headers too
        if ((int64_t)e->h_sc.p->bytes64 > ENC_LIMIT / 2) return too_big();
        RAPID_CHECK(exclusive_scan_i32(epos, n, e->scan_sums, &e->sc.p->alert_bytes, s, nullptr));      // in place: esz -> epos
        RAPID_CHECK(exclusive_scan_i32_to(head, bpos, n, e->scan_sums, s));
        k_enc_batch_sizes<<<grid_for(n), TB, 0, s>>>(n, in.obs, head, bpos, epos, e->sc.p, t, wrap, start, hlen, msz);
        RAPID_KERNEL_CHECK();
        // one batch per sender: the exclusive count of openers at the last alert, plus whether it opens one
        int32_t last[2] = {0, 0};
        RAPID_CUDA(cudaMemcpyAsync(&last[0], bpos + n - 1, 4, cudaMemcpyDeviceToHost, s));
        RAPID_CUDA(cudaMemcpyAsync(&last[1], head + n - 1, 4, cudaMemcpyDeviceToHost, s));
        RAPID_CUDA(cudaStreamSynchronize(s));
        nb = last[0] + last[1];
        RAPID_CHECK(o.hoff.reserve((size_t)nb + 1)); RAPID_CHECK(o.bid.reserve((size_t)nb)); RAPID_CHECK(o.snd.reserve((size_t)nb));
        RAPID_CHECK(e->ids.reserve((size_t)nb));
        int32_t* hpos = e->ids.p;
        RAPID_CHECK(exclusive_scan_i32(hpos, nb, e->scan_sums, &e->sc.p->hdr_bytes, s, nullptr, msz));
        RAPID_CHECK(enc_read_scal(e, s));
        hbytes = e->h_sc.p->hdr_bytes;
        RAPID_CHECK(o.hdr.reserve((size_t)std::max<int64_t>(hbytes, 1)));
        k_enc_batch_emit<<<grid_for(nb), TB, 0, s>>>((int32_t)nb, start, hlen, msz, hpos, in.obs, t, wrap, o.snd.p, o.hdr.p);
        k_enc_alert_emit<<<grid_for(n), TB, 0, s>>>(a, t, head, bpos, epos, start, hlen, hpos, o.hdr.p);
        k_enc_off64<<<grid_for(nb + 1), TB, 0, s>>>((int32_t)nb, hpos, &e->sc.p->hdr_bytes, o.hoff.p);
        k_enc_fill<<<grid_for(nb), TB, 0, s>>>((int32_t)nb, -1, o.bid.p);
        RAPID_KERNEL_CHECK();
    } else {
        RAPID_CUDA(cudaMemsetAsync(o.hoff.p, 0, sizeof(int64_t), s));
    }
    RAPID_CUDA(cudaMemsetAsync(o.boff.p, 0, sizeof(int64_t), s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    o.n = nb; o.n_bodies = 0; o.hdr_bytes = hbytes; o.body_bytes = 0;
    e->cur = 1 - e->cur;
    return RAPID_OK;
}


// Groups the slots' lists (group_proposals): the body of slot s is cls[s], bodies numbered by their lowest slot.  Every entry is
// >= 2 bytes: an encode whose bodies would list more than ENC_LIMIT / 2 entries is refused before they are listed.
template <typename Src>
static int32_t group_bodies(WireEnc* e, cudaStream_t s, int64_t n, const Src& src) {
    RAPID_CHECK(e->cls.reserve((size_t)std::max<int64_t>(n, 1)));
    RAPID_CHECK(group_proposals(s, n, src, e->grp, e->cls.p));
    if ((int64_t)e->grp.h_sc.p->entries64 > ENC_LIMIT / 2) return too_big();
    return RAPID_OK;
}

// The messages of the sending slots of L, in slot order, once group_bodies has run and every body's list is in e->ids at its
// class's offset: bodies first (one thread per entry), then one header per message.
static int32_t encode_lists(WireEnc* e, const WireEncCtx& ctx, const ListIn& L) {
    cudaStream_t s = ctx.stream;
    EncOut& o = e->out[1 - e->cur];
    const int32_t n = L.n;
    const EpTab t = ep_tab(ctx.view);
    const ProposalGroups& g = e->grp;
    const int32_t nb = g.h_sc.p->n_classes, nE = g.h_sc.p->n_entries;
    int32_t *send = g.rep.p, *mpos = g.rpos.p, *hsz = g.loff.p, *hpos = g.slot.p;   // the grouping's per-slot scratch is free
    RAPID_CUDA(cudaMemsetAsync(e->sc.p, 0, sizeof(EncScal), s));
    k_enc_send<<<grid_for(n), TB, 0, s>>>(L, send);
    RAPID_KERNEL_CHECK();
    RAPID_CHECK(exclusive_scan_i32(mpos, n, e->scan_sums, &e->sc.p->n_msgs, s, nullptr, send));
    if (nb > 0) {
        RAPID_CHECK(e->epos.reserve((size_t)nE));
        k_enc_entry_sizes<<<grid_for(nE), TB, 0, s>>>(nE, e->ids.p, t, e->epos.p, e->sc.p);
        RAPID_KERNEL_CHECK();
    }
    RAPID_CHECK(enc_read_scal(e, s));
    if ((int64_t)e->h_sc.p->bytes64 > ENC_LIMIT) return too_big();
    const int64_t nm = e->h_sc.p->n_msgs, bbytes = (int64_t)e->h_sc.p->bytes64;
    int64_t hbytes = 0;
    if (nb > 0) {
        RAPID_CHECK(exclusive_scan_i32(e->epos.p, nE, e->scan_sums, &e->sc.p->body_bytes, s, nullptr));
        RAPID_CHECK(o.bodies.reserve((size_t)std::max<int64_t>(bbytes, 1))); RAPID_CHECK(o.boff.reserve((size_t)nb + 1));
        k_enc_entry_emit<<<grid_for(nE), TB, 0, s>>>(nE, e->ids.p, t, list_tag(L.kind), e->epos.p, o.bodies.p);
        k_enc_body_off<<<grid_for(nb + 1), TB, 0, s>>>(nb, g.c_off.p, e->epos.p, e->sc.p, o.boff.p);
        RAPID_KERNEL_CHECK();
    } else {
        RAPID_CUDA(cudaMemsetAsync(o.boff.p, 0, sizeof(int64_t), s));
    }
    if (nm > 0) {
        RAPID_CHECK(o.hoff.reserve((size_t)nm + 1)); RAPID_CHECK(o.bid.reserve((size_t)nm)); RAPID_CHECK(o.snd.reserve((size_t)nm));
        k_enc_list_sizes<<<grid_for(n), TB, 0, s>>>(L, t, send, mpos, e->cls.p, o.boff.p, hsz);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(exclusive_scan_i32(hpos, nm, e->scan_sums, &e->sc.p->hdr_bytes, s, nullptr, hsz));
        RAPID_CHECK(enc_read_scal(e, s));
        hbytes = e->h_sc.p->hdr_bytes;
        RAPID_CHECK(o.hdr.reserve((size_t)std::max<int64_t>(hbytes, 1)));
        k_enc_list_emit<<<grid_for(n), TB, 0, s>>>(L, t, send, mpos, e->cls.p, o.boff.p, hpos, o.bid.p, o.snd.p, o.hdr.p);
        k_enc_off64<<<grid_for(nm + 1), TB, 0, s>>>((int32_t)nm, hpos, &e->sc.p->hdr_bytes, o.hoff.p);
        RAPID_KERNEL_CHECK();
    } else {
        RAPID_CUDA(cudaMemsetAsync(o.hoff.p, 0, sizeof(int64_t), s));
    }
    RAPID_CUDA(cudaStreamSynchronize(s));
    o.n = nm; o.n_bodies = nb; o.hdr_bytes = hbytes; o.body_bytes = bbytes;
    e->cur = 1 - e->cur;
    return RAPID_OK;
}

// the list cache follows the view's members: ids are renumbered by a cut
static void lists_sync(WireEnc* e, const View* v) {
    if (e->lists_epoch != v->member_epoch) { e->lists.clear(); e->lists_epoch = v->member_epoch; }
}

// a detector receiver's announced proposal in canonical order, checked against the fingerprint it must have
static int32_t cd_list(const rapid_cd* cd, int64_t receiver, uint64_t h1, uint64_t h2, int32_t len, std::vector<int32_t>& ids) {
    ids.assign((size_t)std::max(len, 1), 0);
    int32_t got = 0;
    RAPID_CHECK(rapid_cd_get_proposal(cd, receiver, ids.data(), len, &got));
    uint64_t a = 0, b = 0;
    if (got == len) RAPID_CHECK(rapid_proposal_fingerprint(ids.data(), got, &a, &b));
    if (got != len || a != h1 || b != h2) return -1;
    ids.resize((size_t)len);
    return RAPID_OK;
}

// The votes' bodies: the detector's lists of the grouped proposals (list_proposals, into the encoder's storage: the handle's
// census stays as it was), each checked against its fingerprint and kept in the list cache for the answers.
static int32_t vote_lists(WireEnc* e, cudaStream_t s, const rapid_cd* cd) {
    const ProposalGroups& g = e->grp;
    const int32_t nb = g.h_sc.p->n_classes, nE = g.h_sc.p->n_entries;
    if (nb == 0) return RAPID_OK;
    RAPID_CHECK(e->ids.reserve((size_t)nE));
    RAPID_CHECK(list_proposals(s, cd, e->grp, e->ids.p, nullptr));
    const size_t B = (size_t)nb;
    std::vector<uint64_t> h1(B), h2(B);
    std::vector<int32_t> len(B), fill(B), rep(B), off(B), ids((size_t)nE);
    RAPID_CUDA(cudaMemcpyAsync(h1.data(), g.c_h1.p, B * 8, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaMemcpyAsync(h2.data(), g.c_h2.p, B * 8, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaMemcpyAsync(len.data(), g.c_len.p, B * 4, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaMemcpyAsync(fill.data(), g.c_fill.p, B * 4, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaMemcpyAsync(rep.data(), g.c_rep.p, B * 4, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaMemcpyAsync(off.data(), g.c_off.p, B * 4, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaMemcpyAsync(ids.data(), e->ids.p, (size_t)nE * 4, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    for (size_t b = 0; b < B; ++b) {
        const int32_t* l = ids.data() + off[b];
        uint64_t a = 0, c = 0;
        if (fill[b] == len[b]) RAPID_CHECK(rapid_proposal_fingerprint(l, len[b], &a, &c));
        if (fill[b] != len[b] || a != h1[b] || c != h2[b]) { set_error("receiver %d's proposal does not match its fingerprint", rep[b]); return RAPID_EINVAL; }
        e->lists[std::make_tuple(h1[b], h2[b], len[b])].assign(l, l + len[b]);
    }
    return RAPID_OK;
}

// The answers' bodies: each distinct list from the cache, else from the detector receiver with the representative's index
static int32_t answer_lists(WireEnc* e, cudaStream_t s, const ListIn& L, const rapid_cd* cd) {
    const ProposalGroups& g = e->grp;
    const int32_t nb = g.h_sc.p->n_classes, nE = g.h_sc.p->n_entries;
    if (nb == 0) return RAPID_OK;
    const size_t B = (size_t)nb;
    std::vector<uint64_t> h1(B), h2(B);
    std::vector<int32_t> len(B), rep(B), ids, one;
    RAPID_CUDA(cudaMemcpyAsync(h1.data(), g.c_h1.p, B * 8, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaMemcpyAsync(h2.data(), g.c_h2.p, B * 8, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaMemcpyAsync(len.data(), g.c_len.p, B * 4, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaMemcpyAsync(rep.data(), g.c_rep.p, B * 4, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    ids.reserve((size_t)nE);
    for (size_t b = 0; b < B; ++b) {
        const auto key = std::make_tuple(h1[b], h2[b], len[b]);
        auto it = e->lists.find(key);
        if (it == e->lists.end()) {
            int32_t acc = 0;
            RAPID_CUDA(cudaMemcpyAsync(&acc, L.acc + rep[b], sizeof(int32_t), cudaMemcpyDeviceToHost, s));
            RAPID_CUDA(cudaStreamSynchronize(s));
            const int64_t r = cd ? acc - cd->rbegin : -1;
            if (!cd || r < 0 || r >= cd->R || cd_list(cd, r, h1[b], h2[b], len[b], one) != RAPID_OK) {
                set_error("the %d-endpoint list held by acceptor %lld is not known: encode the votes that carried it first, or pass the "
                          "detector whose receiver announced it", len[b], (long long)acc);
                return RAPID_EINVAL;
            }
            it = e->lists.emplace(key, one).first;
        }
        ids.insert(ids.end(), it->second.begin(), it->second.end());
    }
    RAPID_CHECK(e->ids.reserve((size_t)nE));
    RAPID_CUDA(cudaMemcpyAsync(e->ids.p, ids.data(), (size_t)nE * 4, cudaMemcpyHostToDevice, s));
    return RAPID_OK;
}

static int32_t check_cd(const WireEncCtx& ctx, const rapid_cd* cd) {
    if (cd->view != ctx.view || cd->device != ctx.device) { set_error("the detector was created on another view or device"); return RAPID_EINVAL; }
    if (cd->raw) { set_error("RAW detectors do not announce proposals"); return RAPID_EINVAL; }
    if (cd->member_epoch != ctx.view->member_epoch) { set_error("the view's members changed since the detector was created"); return RAPID_EINVAL; }
    return RAPID_OK;
}

// Phase1b (want = 1) / Phase2b (want = 2) answers of the acceptors
static int32_t encode_answers(rapid_wire* w, const rapid_pxa* pxa, const rapid_cd* cd, uint32_t flags, int want, int64_t* n_messages,
                              int64_t* n_bodies) {
    if (!w || !pxa || (flags & ~RAPID_WIRE_REQUEST)) { set_error("bad arguments"); return RAPID_EINVAL; }
    WireEncCtx ctx;
    wire_enc_ctx(w, &ctx);
    PxaAnswers in;
    pxa_answers_dev(pxa, &in);
    if (in.device != ctx.device) { set_error("the acceptors live on another device"); return RAPID_EINVAL; }
    if (in.kind != want) {
        set_error(want == 1 ? "no Phase1b answers pending (call rapid_pxa_phase1a first)" : "no Phase2b answers pending (call rapid_pxa_phase2a first)");
        return RAPID_EINVAL;
    }
    if (in.begin + in.R > ctx.view->n) { set_error("the acceptors' ring-0 positions exceed the view"); return RAPID_EINVAL; }
    if (cd) RAPID_CHECK(check_cd(ctx, cd));
    DeviceGuard g(ctx.device);
    if (cd) RAPID_CHECK(cd_wait(cd, false));
    WireEnc* e = nullptr;
    RAPID_CHECK(enc_get(w, &ctx, &e));
    lists_sync(e, ctx.view);
    ListIn L{};
    L.n = (int32_t)in.n; L.kind = want == 1 ? RAPID_WIRE_PHASE1B : RAPID_WIRE_PHASE2B; L.wrap = (flags & RAPID_WIRE_REQUEST) ? 1 : 0;
    L.cfg = in.cfg; L.acc = in.sender; L.ring0 = ctx.view->ring.p; L.rank = in.rank;
    if (want == 1) L.vrnd = in.vrnd;
    const AnswerFp fp = want == 1 ? AnswerFp{in.h1, in.h2, in.len, 0, 0, 0} : AnswerFp{nullptr, nullptr, nullptr, in.v_h1, in.v_h2, in.v_len};
    RAPID_CHECK(group_bodies(e, ctx.stream, L.n, fp));
    RAPID_CHECK(answer_lists(e, ctx.stream, L, cd));
    RAPID_CHECK(encode_lists(e, ctx, L));
    const EncOut& o = e->out[e->cur];
    if (n_messages) *n_messages = o.n;
    if (n_bodies) *n_bodies = o.n_bodies;
    return RAPID_OK;
}

}  // namespace rapid

using namespace rapid;

extern "C" {

int32_t rapid_wire_encode_alert_batches(rapid_wire* w, const rapid_fdet* fd, uint32_t flags, int64_t* n_messages, int64_t* n_bytes) {
    if (!w || !fd || (flags & ~RAPID_WIRE_REQUEST)) { set_error("bad arguments"); return RAPID_EINVAL; }
    WireEncCtx ctx;
    wire_enc_ctx(w, &ctx);
    FdetInterval in;
    fdet_interval_dev(fd, &in);
    if (in.view != ctx.view || in.device != ctx.device) { set_error("the failure detectors were created on another view or device"); return RAPID_EINVAL; }
    if (!in.have) { set_error("no failure-detector interval since the last reset (call rapid_fdet_tick first)"); return RAPID_EINVAL; }
    DeviceGuard g(ctx.device);
    WireEnc* e = nullptr;
    RAPID_CHECK(enc_get(w, &ctx, &e));
    RAPID_CHECK(encode_alerts(e, ctx, in, flags));
    const EncOut& o = e->out[e->cur];
    if (n_messages) *n_messages = o.n;
    if (n_bytes) *n_bytes = o.hdr_bytes + o.body_bytes;
    return RAPID_OK;
}

int32_t rapid_wire_encode_votes(rapid_wire* w, const rapid_cd* cd, int64_t cfg_id, uint32_t flags, int64_t* n_messages, int64_t* n_bodies) {
    if (!w || !cd || (flags & ~RAPID_WIRE_REQUEST)) { set_error("bad arguments"); return RAPID_EINVAL; }
    WireEncCtx ctx;
    wire_enc_ctx(w, &ctx);
    RAPID_CHECK(check_cd(ctx, cd));
    if (cd->batch_serial == 0) { set_error("the detector has applied no batch: it has no outputs to encode"); return RAPID_EINVAL; }
    DeviceGuard g(ctx.device);
    RAPID_CHECK(cd_wait(cd, false));                                         // asynchronous batches still in flight on its stream
    WireEnc* e = nullptr;
    RAPID_CHECK(enc_get(w, &ctx, &e));
    lists_sync(e, ctx.view);
    ListIn L{};
    L.n = (int32_t)cd->R; L.kind = RAPID_WIRE_FAST_ROUND_PHASE2B; L.wrap = (flags & RAPID_WIRE_REQUEST) ? 1 : 0; L.cfg = cfg_id;
    L.rflags = cd->rflags.p; L.rbegin = cd->rbegin; L.ring0 = ctx.view->ring.p;
    RAPID_CHECK(group_bodies(e, ctx.stream, L.n, AnnouncedFp{cd->rflags.p, cd->out_h1.p, cd->out_h2.p, cd->out_len.p, 1}));
    RAPID_CHECK(vote_lists(e, ctx.stream, cd));
    RAPID_CHECK(encode_lists(e, ctx, L));
    const EncOut& o = e->out[e->cur];
    if (n_messages) *n_messages = o.n;
    if (n_bodies) *n_bodies = o.n_bodies;
    return RAPID_OK;
}

int32_t rapid_wire_encode_phase1b(rapid_wire* w, const rapid_pxa* pxa, const rapid_cd* cd, uint32_t flags, int64_t* n_messages,
                                  int64_t* n_bodies) {
    return encode_answers(w, pxa, cd, flags, 1, n_messages, n_bodies);
}

int32_t rapid_wire_encode_phase2b(rapid_wire* w, const rapid_pxa* pxa, const rapid_cd* cd, uint32_t flags, int64_t* n_messages,
                                  int64_t* n_bodies) {
    return encode_answers(w, pxa, cd, flags, 2, n_messages, n_bodies);
}

int32_t rapid_wire_encoded_counts(const rapid_wire* cw, int64_t* n_messages, int64_t* header_bytes, int64_t* n_bodies, int64_t* body_bytes) {
    if (!cw) { set_error("NULL handle"); return RAPID_EINVAL; }
    WireEncCtx ctx;
    wire_enc_ctx(const_cast<rapid_wire*>(cw), &ctx);
    const EncOut* o = *ctx.enc ? &(*ctx.enc)->out[(*ctx.enc)->cur] : nullptr;
    if (n_messages) *n_messages = o ? o->n : 0;
    if (header_bytes) *header_bytes = o ? o->hdr_bytes : 0;
    if (n_bodies) *n_bodies = o ? o->n_bodies : 0;
    if (body_bytes) *body_bytes = o ? o->body_bytes : 0;
    return RAPID_OK;
}

int32_t rapid_wire_encoded_dev(const rapid_wire* cw, const uint8_t** headers, const int64_t** header_off, const int32_t** body_id,
                               const uint8_t** bodies, const int64_t** body_off) {
    if (!cw) { set_error("NULL handle"); return RAPID_EINVAL; }
    WireEncCtx ctx;
    wire_enc_ctx(const_cast<rapid_wire*>(cw), &ctx);
    if (!*ctx.enc) { set_error("nothing was encoded on this handle"); return RAPID_EINVAL; }
    const EncOut& o = (*ctx.enc)->out[(*ctx.enc)->cur];
    if (headers) *headers = o.hdr.p;
    if (header_off) *header_off = o.hoff.p;
    if (body_id) *body_id = o.bid.p;
    if (bodies) *bodies = o.bodies.p;
    if (body_off) *body_off = o.boff.p;
    return RAPID_OK;
}

int32_t rapid_wire_read_encoded(const rapid_wire* cw, uint8_t* headers, int64_t* header_off, int32_t* body_id, uint8_t* bodies,
                                int64_t* body_off) {
    if (!cw) { set_error("NULL handle"); return RAPID_EINVAL; }
    WireEncCtx ctx;
    wire_enc_ctx(const_cast<rapid_wire*>(cw), &ctx);
    if (!*ctx.enc) { set_error("nothing was encoded on this handle"); return RAPID_EINVAL; }
    const EncOut& o = (*ctx.enc)->out[(*ctx.enc)->cur];
    DeviceGuard g(ctx.device);
    cudaStream_t s = ctx.stream;
    if (headers && o.hdr_bytes) RAPID_CUDA(cudaMemcpyAsync(headers, o.hdr.p, (size_t)o.hdr_bytes, cudaMemcpyDeviceToHost, s));
    if (header_off) RAPID_CUDA(cudaMemcpyAsync(header_off, o.hoff.p, ((size_t)o.n + 1) * 8, cudaMemcpyDeviceToHost, s));
    if (body_id && o.n) RAPID_CUDA(cudaMemcpyAsync(body_id, o.bid.p, (size_t)o.n * 4, cudaMemcpyDeviceToHost, s));
    if (bodies && o.body_bytes) RAPID_CUDA(cudaMemcpyAsync(bodies, o.bodies.p, (size_t)o.body_bytes, cudaMemcpyDeviceToHost, s));
    if (body_off) RAPID_CUDA(cudaMemcpyAsync(body_off, o.boff.p, ((size_t)o.n_bodies + 1) * 8, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

int32_t rapid_wire_read_encoded_sizes(const rapid_wire* cw, int64_t* sizes) {
    if (!cw) { set_error("NULL handle"); return RAPID_EINVAL; }
    WireEncCtx ctx;
    wire_enc_ctx(const_cast<rapid_wire*>(cw), &ctx);
    if (!*ctx.enc) { set_error("nothing was encoded on this handle"); return RAPID_EINVAL; }
    WireEnc* e = *ctx.enc;
    const EncOut& o = e->out[e->cur];
    if (o.n == 0) return RAPID_OK;
    if (!sizes) { set_error("NULL sizes"); return RAPID_EINVAL; }
    DeviceGuard g(ctx.device);
    cudaStream_t s = ctx.stream;
    RAPID_CHECK(e->sizes.reserve((size_t)o.n));
    k_enc_sizes<<<grid_for(o.n), TB, 0, s>>>(o.n, o.hoff.p, o.bid.p, o.boff.p, e->sizes.p);
    RAPID_KERNEL_CHECK();
    RAPID_CUDA(cudaMemcpyAsync(sizes, e->sizes.p, (size_t)o.n * 8, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

int32_t rapid_wire_read_encoded_senders(const rapid_wire* cw, int32_t* sender) {
    if (!cw) { set_error("NULL handle"); return RAPID_EINVAL; }
    WireEncCtx ctx;
    wire_enc_ctx(const_cast<rapid_wire*>(cw), &ctx);
    if (!*ctx.enc) { set_error("nothing was encoded on this handle"); return RAPID_EINVAL; }
    const EncOut& o = (*ctx.enc)->out[(*ctx.enc)->cur];
    if (o.n == 0) return RAPID_OK;
    if (!sender) { set_error("NULL sender"); return RAPID_EINVAL; }
    DeviceGuard g(ctx.device);
    RAPID_CUDA(cudaMemcpyAsync(sender, o.snd.p, (size_t)o.n * 4, cudaMemcpyDeviceToHost, ctx.stream));
    RAPID_CUDA(cudaStreamSynchronize(ctx.stream));
    return RAPID_OK;
}

}  // extern "C"
