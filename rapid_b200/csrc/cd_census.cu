// Proposal census (DESIGN §4.15): the distinct proposals announced by a cut detector's receivers in its last call, each with
// its voters, its lowest receiver, its list in canonical ring-0 order with a status per entry (VIEW_CHANGE_PROPOSAL's
// NodeStatusChange list, MembershipService.java:336-345, :586-593) and, given a cut, how many of its entries the cut holds.
//
//   claim     one thread per receiver: every announcer inserts its (h1, h2, len) into an open-addressing table (fp_table_claim);
//             a slot keeps the lowest receiver and counts its voters
//   classes   representatives (the lowest receiver of a fingerprint) marked and scanned: class c is the c-th representative in
//             receiver order; cls[r] = class of receiver r, -1 if r did not announce; list offsets are the scan of the
//             representatives' lengths
//   lists     one thread per (class, subject slot) tests the representative's row with rapid_cd_get_proposal's rule
//             (in_announced_proposal), then three stable LSD radix sorts over all entries at once — by id, by the sign-flipped
//             ring-0 key, by class — give every list get_proposal's order
//   status    DOWN for a member id, UP for a registered joiner (createNodeStatusChangeList :586-593)
//   in_cut    one block per class counts its entries in a device bitmap of the cut
// Claim and classes (group_proposals) and the lists (list_proposals) are also the wire encoder's (wire_encode.cu): it groups its
// votes' and answers' lists with them, in storage of its own.  One host synchronisation per census: the class and entry counts
// the caller gets back, which also size the per-class arrays and the sorts.  The lists are enqueued after it on the handle's
// stream; the reads wait for them.  Outputs are double-buffered: a census writes the spare set and swaps on success, so a
// refused or failed census leaves the previous one as it was.
#include <algorithm>
#include <vector>

#include "cd_internal.cuh"
#include "radix.cuh"
#include "scan.cuh"

namespace rapid {

struct CensusOut {
    bool valid = false;
    int64_t n_classes = 0, n_entries = 0;
    DevBuf<uint64_t> h1, h2;           // [n_classes]
    DevBuf<int32_t> len, voters, rep, in_cut;
    DevBuf<int64_t> off;               // [n_classes + 1]
    DevBuf<int32_t> ids;               // [n_entries]
    DevBuf<uint8_t> status;
    DevBuf<int32_t> cls;               // [R]
};

struct Census {
    CensusOut out[2];
    int cur = 0;                       // out[cur] holds the last census
    ProposalGroups g;
    DevBuf<int32_t> cut_ids;
    DevBuf<uint32_t> cut_bits;
};

// the lists stage's scratch: per entry, and the sorts'
struct ListScratch {
    DevBuf<int32_t> e_id, e_cls, idx, k32, k32s, perm;                // [n_entries]
    DevBuf<uint64_t> e_key, k64, k64s;
    RadixScratch rs;
};

ProposalGroups::~ProposalGroups() { delete ls; }

void census_destroy(CD* cd) {
    delete cd->census;
    cd->census = nullptr;
}

static const int TB = 256;
static inline unsigned grid_for(int64_t n) { return (unsigned)ceil_div<int64_t>(n > 0 ? n : 1, TB); }
constexpr int CEN_TABLE_MIN = 1024;
constexpr uint64_t KEY_SIGN = 0x8000000000000000ULL;   // signed ring-0 key -> unsigned order

// ------------------------------------------------------------------ claim and classes
template <typename Src>
__global__ void k_cen_count(int64_t n, Src src, GroupScal* __restrict__ sc) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool part = i < n && src.part((int32_t)i);
    const unsigned b = __ballot_sync(0xffffffffu, part);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(&sc->n_part, __popc(b));
}

// T = the smallest power of two >= 2 x items taking part (at least CEN_TABLE_MIN), chosen on the device; grid-stride fill of T slots
__global__ void k_cen_table_init(GroupScal* __restrict__ sc, int32_t* __restrict__ table, int32_t* __restrict__ tcnt) {
    uint32_t T = CEN_TABLE_MIN;
    while ((int64_t)T < 2 * (int64_t)sc->n_part) T <<= 1;
    if (blockIdx.x == 0 && threadIdx.x == 0) sc->T = (int32_t)T;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < T; i += gridDim.x * blockDim.x) { table[i] = -1; tcnt[i] = 0; }
}

template <typename Src>
__global__ void k_cen_claim(int64_t n, Src src, const GroupScal* __restrict__ sc, int32_t* __restrict__ table,
                            int32_t* __restrict__ tcnt, int32_t* __restrict__ slot) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (!src.part((int32_t)i)) { slot[i] = -1; return; }
    uint64_t a, b; int32_t l;
    src((int32_t)i, &a, &b, &l);
    const uint32_t pos = fp_table_claim(table, (uint32_t)sc->T, (int32_t)i, a, b, l, src);
    atomicAdd(&tcnt[pos], 1);
    slot[i] = (int32_t)pos;
}

// rep[i]: i is its fingerprint's lowest item; loff[i]: its list length if so (scanned into list offsets)
template <typename Src>
__global__ void k_cen_rep(int64_t n, Src src, const int32_t* __restrict__ slot, const int32_t* __restrict__ table,
                          int32_t* __restrict__ rep, int32_t* __restrict__ loff, GroupScal* __restrict__ sc) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool is = slot[i] >= 0 && table[slot[i]] == (int32_t)i;
    const int32_t l = is ? src.length((int32_t)i) : 0;
    rep[i] = is ? 1 : 0;
    loff[i] = l;
    if (is) atomicAdd(&sc->entries64, (unsigned long long)l);
}

template <typename Src>
struct ClassArgs {
    int64_t n;
    const int32_t* slot;
    const int32_t* table;
    const int32_t* tcnt;
    const int32_t* rep;
    const int32_t* rpos;
    const int32_t* loff;
    Src src;
    int32_t* cls;
    uint64_t* c_h1;
    uint64_t* c_h2;
    int32_t *c_rep, *c_len, *c_voters, *c_off;
};
template <typename Src>
__global__ void k_cen_classes(ClassArgs<Src> a) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    const int32_t sl = a.slot[i];
    a.cls[i] = sl >= 0 ? a.rpos[a.table[sl]] : -1;
    if (!a.rep[i]) return;
    const int32_t c = a.rpos[i];
    a.src((int32_t)i, &a.c_h1[c], &a.c_h2[c], &a.c_len[c]);
    a.c_rep[c] = (int32_t)i;
    a.c_voters[c] = a.tcnt[sl];
    a.c_off[c] = a.loff[i];
}

// ------------------------------------------------------------------ lists
__global__ void k_cen_class_out(int32_t nc, int32_t ne, const uint64_t* __restrict__ c_h1, const uint64_t* __restrict__ c_h2,
                                const int32_t* __restrict__ c_len, const int32_t* __restrict__ c_voters, const int32_t* __restrict__ c_rep,
                                const int32_t* __restrict__ c_off, uint64_t* __restrict__ h1, uint64_t* __restrict__ h2,
                                int32_t* __restrict__ len, int32_t* __restrict__ voters, int32_t* __restrict__ rep, int64_t* __restrict__ off) {
    const int32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c == nc) off[c] = ne;
    if (c >= nc) return;
    h1[c] = c_h1[c]; h2[c] = c_h2[c]; len[c] = c_len[c]; voters[c] = c_voters[c]; rep[c] = c_rep[c];
    off[c] = c_off[c];
}

// one thread per (class, subject slot): the slot's subject joins the class's list if its representative announced it.  Lanes of a
// warp that add to the same class take their places with one atomic (__match_any_sync); the order inside a class is settled by
// the sorts.  A class never takes more than its length (a guard: the rule lists exactly len entries).
struct GatherArgs {
    int32_t nc, S, H;
    uint32_t RM;
    RowRef rows;
    MarkPlane emit;
    const uint32_t* rflags;
    const int32_t* c_rep;
    const int32_t* c_off;
    const int32_t* c_len;
    int32_t* c_fill;
    const int32_t* slot_subject;
    const int64_t* key0;
    int32_t* e_id;
    int32_t* e_cls;
    uint64_t* e_key;
};
__global__ void k_cen_gather(GatherArgs a) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = (int64_t)a.nc * a.S;
    const int32_t c = i < n ? (int32_t)(i / a.S) : -1;
    const int32_t s = i < n ? (int32_t)(i - (int64_t)c * a.S) : 0;
    const int32_t r = i < n ? a.c_rep[c] : 0;
    const bool in = i < n && in_announced_proposal(a.rows, a.emit, s, r, a.H, a.RM, (a.rflags[r] & RF_RULE_GE_H) ? 1 : 0);
    const unsigned act = __ballot_sync(0xffffffffu, in);
    if (!in) return;
    const unsigned peers = __match_any_sync(act, c);
    const int lane = threadIdx.x & 31, leader = __ffs(peers) - 1;
    int32_t base = 0;
    if (lane == leader) base = atomicAdd(&a.c_fill[c], __popc(peers));
    base = __shfl_sync(peers, base, leader);
    const int32_t k = base + __popc(peers & ((1u << lane) - 1u));
    if (k >= a.c_len[c]) return;
    const int32_t at = a.c_off[c] + k;
    const int32_t id = a.slot_subject[s];
    a.e_id[at] = id;
    a.e_cls[at] = c;
    a.e_key[at] = (uint64_t)a.key0[id] ^ KEY_SIGN;
}

__global__ void k_cen_iota(int32_t n, const int32_t* __restrict__ e_id, int32_t* __restrict__ k32, int32_t* __restrict__ idx) {
    const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) { k32[j] = e_id[j]; idx[j] = j; }
}
// the next pass's keys in the current order of the entries
__global__ void k_cen_key64(int32_t n, const int32_t* __restrict__ perm, const uint64_t* __restrict__ e_key, uint64_t* __restrict__ k) {
    const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) k[j] = e_key[perm[j]];
}
__global__ void k_cen_key32(int32_t n, const int32_t* __restrict__ perm, const int32_t* __restrict__ src, int32_t* __restrict__ k) {
    const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) k[j] = src[perm[j]];
}
__global__ void k_cen_entries(int32_t n, int64_t members, const int32_t* __restrict__ perm, const int32_t* __restrict__ e_id,
                              int32_t* __restrict__ ids, uint8_t* __restrict__ status) {
    const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int32_t id = e_id[perm[j]];
    ids[j] = id;
    if (status) status[j] = id < members ? RAPID_EDGE_DOWN : RAPID_EDGE_UP;
}

// ------------------------------------------------------------------ distance from a cut
__global__ void k_cen_cut_bits(int32_t n, const int32_t* __restrict__ ids, uint32_t* __restrict__ bits) {
    const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) atomicOr(&bits[ids[j] >> 5], 1u << (ids[j] & 31));
}
// block c: entries of class c in the cut
__global__ void __launch_bounds__(TB) k_cen_in_cut(const int64_t* __restrict__ off, const int32_t* __restrict__ ids,
                                                   const uint32_t* __restrict__ bits, int32_t* __restrict__ in_cut) {
    __shared__ int32_t warp_sums[TB / 32];
    const int32_t c = blockIdx.x;
    int32_t k = 0;
    for (int64_t j = off[c] + threadIdx.x; j < off[c + 1]; j += TB) k += (bits[ids[j] >> 5] >> (ids[j] & 31)) & 1u;
    int32_t total;
    scan_block_exclusive(k, warp_sums, &total);
    if (threadIdx.x == 0) in_cut[c] = total;
}

// ------------------------------------------------------------------ host side
template <typename Src>
int32_t group_proposals(cudaStream_t s, int64_t n, const Src& src, ProposalGroups& g, int32_t* cls) {
    const size_t N = (size_t)std::max<int64_t>(n, 1);
    uint32_t Tcap = CEN_TABLE_MIN;
    while ((int64_t)Tcap < 2 * n) Tcap <<= 1;
    RAPID_CHECK(g.sc.reserve(1)); RAPID_CHECK(g.h_sc.reserve(1));
    RAPID_CHECK(g.table.reserve(Tcap)); RAPID_CHECK(g.tcnt.reserve(Tcap));
    RAPID_CHECK(g.slot.reserve(N)); RAPID_CHECK(g.rep.reserve(N)); RAPID_CHECK(g.rpos.reserve(N)); RAPID_CHECK(g.loff.reserve(N));
    RAPID_CUDA(cudaMemsetAsync(g.sc.p, 0, sizeof(GroupScal), s));
    k_cen_count<<<grid_for(n), TB, 0, s>>>(n, src, g.sc.p);
    k_cen_table_init<<<(unsigned)std::min<int64_t>(ceil_div<int64_t>(Tcap, TB), 4 * TARGET_SMS), TB, 0, s>>>(g.sc.p, g.table.p, g.tcnt.p);
    k_cen_claim<<<grid_for(n), TB, 0, s>>>(n, src, g.sc.p, g.table.p, g.tcnt.p, g.slot.p);
    k_cen_rep<<<grid_for(n), TB, 0, s>>>(n, src, g.slot.p, g.table.p, g.rep.p, g.loff.p, g.sc.p);
    RAPID_KERNEL_CHECK();
    RAPID_CHECK(exclusive_scan_i32(g.rpos.p, n, g.scan_sums, &g.sc.p->n_classes, s, nullptr, g.rep.p));
    RAPID_CHECK(exclusive_scan_i32(g.loff.p, n, g.scan_sums, &g.sc.p->n_entries, s, nullptr));
    RAPID_CUDA(cudaMemcpyAsync(g.h_sc.p, g.sc.p, sizeof(GroupScal), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    const size_t C = (size_t)std::max(g.h_sc.p->n_classes, 1);
    RAPID_CHECK(g.c_h1.reserve(C)); RAPID_CHECK(g.c_h2.reserve(C)); RAPID_CHECK(g.c_rep.reserve(C)); RAPID_CHECK(g.c_len.reserve(C));
    RAPID_CHECK(g.c_voters.reserve(C)); RAPID_CHECK(g.c_off.reserve(C)); RAPID_CHECK(g.c_fill.reserve(C));
    ClassArgs<Src> ca{n, g.slot.p, g.table.p, g.tcnt.p, g.rep.p, g.rpos.p, g.loff.p, src, cls,
                      g.c_h1.p, g.c_h2.p, g.c_rep.p, g.c_len.p, g.c_voters.p, g.c_off.p};
    k_cen_classes<<<grid_for(n), TB, 0, s>>>(ca);
    RAPID_KERNEL_CHECK();
    return RAPID_OK;
}
template int32_t group_proposals<AnnouncedFp>(cudaStream_t, int64_t, const AnnouncedFp&, ProposalGroups&, int32_t*);
template int32_t group_proposals<AnswerFp>(cudaStream_t, int64_t, const AnswerFp&, ProposalGroups&, int32_t*);

static int bits_for(int64_t n) {                  // bits of the largest value below n (at least 1)
    int b = 1;
    while (b < 62 && ((int64_t)1 << b) < n) ++b;
    return b;
}

int32_t list_proposals(cudaStream_t s, const CD* cd, ProposalGroups& g, int32_t* ids, uint8_t* status) {
    const int32_t nc = g.h_sc.p->n_classes, ne = g.h_sc.p->n_entries;
    if (ne <= 0) return RAPID_OK;
    if (!g.ls) g.ls = new ListScratch();
    ListScratch& e = *g.ls;
    const size_t E = (size_t)ne;
    RAPID_CHECK(e.e_id.reserve(E)); RAPID_CHECK(e.e_cls.reserve(E)); RAPID_CHECK(e.e_key.reserve(E));
    RAPID_CHECK(e.idx.reserve(E)); RAPID_CHECK(e.perm.reserve(E)); RAPID_CHECK(e.k32.reserve(E)); RAPID_CHECK(e.k32s.reserve(E));
    RAPID_CHECK(e.k64.reserve(E)); RAPID_CHECK(e.k64s.reserve(E));
    RAPID_CUDA(cudaMemsetAsync(g.c_fill.p, 0, (size_t)nc * sizeof(int32_t), s));
    const int32_t S = cd->S;
    GatherArgs ga{nc, S, cd->H, (1u << cd->K) - 1u, rowref(cd), emit_plane(cd), cd->rflags.p, g.c_rep.p, g.c_off.p, g.c_len.p,
                  g.c_fill.p, cd->slot_subject.p, cd->view->key.p /* ring 0 row */, e.e_id.p, e.e_cls.p, e.e_key.p};
    k_cen_gather<<<grid_for((int64_t)nc * S), TB, 0, s>>>(ga);
    // stable LSD: by id, then by signed ring-0 key, then by class
    k_cen_iota<<<grid_for(ne), TB, 0, s>>>(ne, e.e_id.p, e.k32.p, e.idx.p);
    RAPID_KERNEL_CHECK();
    uint32_t* k32 = reinterpret_cast<uint32_t*>(e.k32.p);
    uint32_t* k32s = reinterpret_cast<uint32_t*>(e.k32s.p);
    RAPID_CHECK(radix_sort_pairs<uint32_t>(e.rs, k32, e.idx.p, k32s, e.perm.p, ne, 0, bits_for(cd->view->n + cd->view->nj), s));
    k_cen_key64<<<grid_for(ne), TB, 0, s>>>(ne, e.perm.p, e.e_key.p, e.k64.p);
    RAPID_KERNEL_CHECK();
    RAPID_CHECK(radix_sort_pairs<uint64_t>(e.rs, e.k64.p, e.perm.p, e.k64s.p, e.idx.p, ne, 0, 64, s));
    int32_t* order = e.idx.p;
    if (nc > 1) {
        k_cen_key32<<<grid_for(ne), TB, 0, s>>>(ne, e.idx.p, e.e_cls.p, e.k32.p);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(radix_sort_pairs<uint32_t>(e.rs, k32, e.idx.p, k32s, e.perm.p, ne, 0, bits_for(nc), s));
        order = e.perm.p;
    }
    k_cen_entries<<<grid_for(ne), TB, 0, s>>>(ne, cd->view->n, order, e.e_id.p, ids, status);
    RAPID_KERNEL_CHECK();
    return RAPID_OK;
}

static int32_t census_run(CD* cd, Census* e, const int32_t* cut_ids, int32_t cut_len) {
    cudaStream_t s = cd->stream;
    CensusOut& o = e->out[1 - e->cur];
    const int64_t R = cd->R;
    const int64_t ntot = cd->view->n + cd->view->nj;
    // the cut's bitmap (ids checked by the caller)
    if (cut_ids) {
        const size_t words = (size_t)ceil_div<int64_t>(std::max<int64_t>(ntot, 1), 32);
        RAPID_CHECK(e->cut_bits.reserve(words)); RAPID_CHECK(e->cut_ids.reserve((size_t)std::max(cut_len, 1)));
        RAPID_CUDA(cudaMemsetAsync(e->cut_bits.p, 0, words * sizeof(uint32_t), s));
        if (cut_len) {
            RAPID_CUDA(cudaMemcpyAsync(e->cut_ids.p, cut_ids, (size_t)cut_len * sizeof(int32_t), cudaMemcpyHostToDevice, s));
            k_cen_cut_bits<<<grid_for(cut_len), TB, 0, s>>>(cut_len, e->cut_ids.p, e->cut_bits.p);
            RAPID_KERNEL_CHECK();
        }
    }
    // ---- claim and classes; the one synchronisation: the counts the caller gets back, which size the lists
    RAPID_CHECK(o.cls.reserve((size_t)R));
    const AnnouncedFp fp{cd->rflags.p, cd->out_h1.p, cd->out_h2.p, cd->out_len.p, 0};
    RAPID_CHECK(group_proposals(s, R, fp, e->g, o.cls.p));
    const GroupScal h = *e->g.h_sc.p;
    if (h.entries64 >= (1ULL << 30)) { set_error("the census would list %llu entries (at most 2^30)", h.entries64); return RAPID_ENOMEM; }
    const int32_t nc = h.n_classes, ne = h.n_entries;
    // ---- lists
    RAPID_CHECK(o.h1.reserve((size_t)std::max(nc, 1))); RAPID_CHECK(o.h2.reserve((size_t)std::max(nc, 1)));
    RAPID_CHECK(o.len.reserve((size_t)std::max(nc, 1))); RAPID_CHECK(o.voters.reserve((size_t)std::max(nc, 1)));
    RAPID_CHECK(o.rep.reserve((size_t)std::max(nc, 1))); RAPID_CHECK(o.in_cut.reserve((size_t)std::max(nc, 1)));
    RAPID_CHECK(o.off.reserve((size_t)nc + 1));
    RAPID_CHECK(o.ids.reserve((size_t)std::max(ne, 1))); RAPID_CHECK(o.status.reserve((size_t)std::max(ne, 1)));
    const ProposalGroups& g = e->g;
    k_cen_class_out<<<grid_for((int64_t)nc + 1), TB, 0, s>>>(nc, ne, g.c_h1.p, g.c_h2.p, g.c_len.p, g.c_voters.p, g.c_rep.p,
                                                             g.c_off.p, o.h1.p, o.h2.p, o.len.p, o.voters.p, o.rep.p, o.off.p);
    RAPID_KERNEL_CHECK();
    RAPID_CHECK(list_proposals(s, cd, e->g, o.ids.p, o.status.p));
    if (nc > 0) {
        if (cut_ids) k_cen_in_cut<<<(unsigned)nc, TB, 0, s>>>(o.off.p, o.ids.p, e->cut_bits.p, o.in_cut.p);
        else RAPID_CUDA(cudaMemsetAsync(o.in_cut.p, 0xff, (size_t)nc * sizeof(int32_t), s));
        RAPID_KERNEL_CHECK();
    }
    RAPID_CUDA(cudaEventRecord(cd->ev_done, s));      // other streams that read the census wait on the handle's event
    o.valid = true;
    o.n_classes = nc;
    o.n_entries = ne;
    e->cur = 1 - e->cur;
    return RAPID_OK;
}

static int32_t census_current(const rapid_cd* cd, const CensusOut** out) {
    if (!cd) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (!cd->census || !cd->census->out[cd->census->cur].valid) { set_error("no proposal census on this handle (call rapid_cd_proposal_census first)"); return RAPID_EINVAL; }
    *out = &cd->census->out[cd->census->cur];
    return RAPID_OK;
}

}  // namespace rapid

using namespace rapid;

extern "C" {

int32_t rapid_cd_proposal_census(rapid_cd* cd, const int32_t* cut_ids, int32_t cut_len, int64_t* n_classes, int64_t* n_entries) {
    if (!cd || cut_len < 0 || (cut_len > 0 && !cut_ids)) { set_error("bad arguments"); return RAPID_EINVAL; }
    if (cd->raw) { set_error("RAW detectors do not announce proposals"); return RAPID_EINVAL; }
    if (cd->batch_serial == 0) { set_error("the detector has applied no batch: it has no announced proposals"); return RAPID_EINVAL; }
    if (cd->member_epoch != cd->view->member_epoch) { set_error("the view's members changed since the detector was created"); return RAPID_EINVAL; }
    if (cut_ids) {
        const int64_t ntot = cd->view->n + cd->view->nj;
        std::vector<int32_t> sorted(cut_ids, cut_ids + cut_len);
        std::sort(sorted.begin(), sorted.end());
        for (int32_t i = 0; i < cut_len; ++i) {
            if (sorted[(size_t)i] < 0 || sorted[(size_t)i] >= ntot) { set_error("cut id %d outside [0, members + registered joiners)", sorted[(size_t)i]); return RAPID_EINVAL; }
            if (i && sorted[(size_t)i] == sorted[(size_t)i - 1]) { set_error("cut id %d appears twice", sorted[(size_t)i]); return RAPID_EINVAL; }
        }
    }
    DeviceGuard g(cd->device);
    RAPID_CHECK(cd_wait(cd, false));      // asynchronous batches still in flight on the handle's stream
    if (!cd->census) cd->census = new Census();
    Census* e = cd->census;
    RAPID_CHECK(census_run(cd, e, cut_ids, cut_len));
    const CensusOut& o = e->out[e->cur];
    if (n_classes) *n_classes = o.n_classes;
    if (n_entries) *n_entries = o.n_entries;
    return RAPID_OK;
}

int32_t rapid_cd_read_census(const rapid_cd* cd, uint64_t* hash, uint64_t* hash2, int32_t* len, int32_t* voters, int32_t* representative,
                             int32_t* in_cut, int64_t* list_off, int32_t* ids, uint8_t* status) {
    const CensusOut* o = nullptr;
    RAPID_CHECK(census_current(cd, &o));
    DeviceGuard g(cd->device);
    cudaStream_t s = cd->stream;
    const size_t nc = (size_t)o->n_classes, ne = (size_t)o->n_entries;
    if (nc) {
        if (hash) RAPID_CUDA(cudaMemcpyAsync(hash, o->h1.p, nc * 8, cudaMemcpyDeviceToHost, s));
        if (hash2) RAPID_CUDA(cudaMemcpyAsync(hash2, o->h2.p, nc * 8, cudaMemcpyDeviceToHost, s));
        if (len) RAPID_CUDA(cudaMemcpyAsync(len, o->len.p, nc * 4, cudaMemcpyDeviceToHost, s));
        if (voters) RAPID_CUDA(cudaMemcpyAsync(voters, o->voters.p, nc * 4, cudaMemcpyDeviceToHost, s));
        if (representative) RAPID_CUDA(cudaMemcpyAsync(representative, o->rep.p, nc * 4, cudaMemcpyDeviceToHost, s));
        if (in_cut) RAPID_CUDA(cudaMemcpyAsync(in_cut, o->in_cut.p, nc * 4, cudaMemcpyDeviceToHost, s));
    }
    if (list_off) RAPID_CUDA(cudaMemcpyAsync(list_off, o->off.p, (nc + 1) * 8, cudaMemcpyDeviceToHost, s));
    if (ne) {
        if (ids) RAPID_CUDA(cudaMemcpyAsync(ids, o->ids.p, ne * 4, cudaMemcpyDeviceToHost, s));
        if (status) RAPID_CUDA(cudaMemcpyAsync(status, o->status.p, ne, cudaMemcpyDeviceToHost, s));
    }
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

int32_t rapid_cd_census_classes_dev(const rapid_cd* cd, const int32_t** cls_dev) {
    const CensusOut* o = nullptr;
    RAPID_CHECK(census_current(cd, &o));
    if (!cls_dev) { set_error("NULL cls_dev"); return RAPID_EINVAL; }
    *cls_dev = o->cls.p;
    return RAPID_OK;
}

int32_t rapid_cd_read_census_classes(const rapid_cd* cd, int32_t* cls) {
    const CensusOut* o = nullptr;
    RAPID_CHECK(census_current(cd, &o));
    if (!cls) { set_error("NULL cls"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    RAPID_CUDA(cudaMemcpyAsync(cls, o->cls.p, (size_t)cd->R * sizeof(int32_t), cudaMemcpyDeviceToHost, cd->stream));
    RAPID_CUDA(cudaStreamSynchronize(cd->stream));
    return RAPID_OK;
}

}  // extern "C"
