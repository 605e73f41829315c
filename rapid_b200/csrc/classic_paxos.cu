// Classic-Paxos fallback (Paxos.java) on the device — SURVEY.md §8 f2.
//
// Three pieces, all integer work over message arrays that live in HBM:
//   * the coordinator rule (selectProposalUsingCoordinatorRule :271-328): max rank -> collect -> distinct values ->
//     "first value whose (N/4+1)-th occurrence comes earliest in arrival order" -> first non-empty fallback;
//   * the coordinator's Phase1b list (:159-191) and the learner's Phase2b sets (:223-236), one node's worth (rapid_px);
//   * the acceptor registers rnd / vrnd / vval of R virtual nodes (:120-151, :198-216, :244-257) (rapid_pxa), whose answers
//     feed the tallies from one handle or, gathered in ascending acceptor_begin, from several shards on one GPU or across ranks.
// "k-th occurrence of a key in arrival order" is the one shared primitive: stable radix sort of (key, arrival index),
// then the element at offset k of each key's run.  Everything is exact; nothing depends on thread scheduling.
#include <limits.h>


#include <algorithm>

#include "cd_internal.cuh"
#include "common.cuh"
#include "nccl_api.cuh"
#include "radix.cuh"
#include "scan.cuh"
#include "wire_internal.cuh"

namespace rapid {

struct PxScal {
    long long max_rank;
    int32_t first_nonempty, first_collected, n_collected, distinct, kth_min, chosen;
    int32_t kept, batch_first_nonempty;          // phase1b append
    int32_t decide_idx, overflow, inserted;      // phase2b
    uint64_t h1, h2;                             // value of `chosen` / of the deciding message
    int32_t len, src;                            // src: batch index of the trigger message
    int32_t unknown_sender;                      // phase2b from the wire: first current-configuration message of an unknown sender
};

// One open-addressing entry = one 32-byte sector: a probe, its key compare and its value update touch a single line.
struct __align__(32) PxEntry {
    int32_t state;       // 0 empty, 1 being published, 2 ready
    int32_t c;
    uint64_t a, b;
    int32_t val;         // pairs: earliest arrival of a new pair (INT_MAX fresh, -1 sealed); round counters: distinct senders so far
    int32_t pad_;
};
struct PxTable {
    uint32_t T;
    PxEntry* e;
};

__device__ __forceinline__ uint32_t px_hash(uint64_t a, uint64_t b, int32_t c) {
    return (uint32_t)(splitmix64(a ^ rotl64(b, 21) ^ ((uint64_t)(uint32_t)c * 0x9E3779B97F4A7C15ULL)) >> 32);
}

// find-or-insert of a 3-word key; -1 when the table is full (the caller reports it)
__device__ int32_t px_find_or_insert(const PxTable t, uint64_t a, uint64_t b, int32_t c, bool* is_new) {
    uint32_t pos = px_hash(a, b, c) & (t.T - 1);
    *is_new = false;
    for (uint32_t probes = 0; probes < t.T; ++probes) {
        int32_t state = *(volatile int32_t*)&t.e[pos].state;
        if (state == 0) state = atomicCAS(&t.e[pos].state, 0, 1);
        if (state == 0) {
            t.e[pos].a = a; t.e[pos].b = b; t.e[pos].c = c;
            __threadfence();
            atomicExch(&t.e[pos].state, 2);
            *is_new = true;
            return (int32_t)pos;
        }
        while (state == 1) state = atomicAdd(&t.e[pos].state, 0);
        __threadfence();
        if (t.e[pos].a == a && t.e[pos].b == b && t.e[pos].c == c) return (int32_t)pos;
        pos = (pos + 1) & (t.T - 1);
    }
    return -1;
}

// Warp-aggregated find-or-insert: one probe per distinct key per warp (a million messages typically carry a handful of
// values, and without this every thread of the first wave fights over the same entry).  EVERY thread of the warp must call
// it; `valid` says whether this lane has a key.  *is_new is set on one lane per newly inserted key.
__device__ int32_t px_find_or_insert_warp(const PxTable t, bool valid, uint64_t a, uint64_t b, int32_t c, bool* is_new) {
    *is_new = false;
    const unsigned active = __ballot_sync(0xffffffffu, valid);
    if (!valid) return -1;
    const unsigned same = __match_any_sync(active, a ^ rotl64(b, 21) ^ ((uint64_t)(uint32_t)c << 1));
    const int leader = __ffs(same) - 1;
    int32_t e = -1;
    bool nw = false;
    if ((int)(threadIdx.x & 31) == leader) e = px_find_or_insert(t, a, b, c, &nw);
    e = __shfl_sync(same, e, leader);
    const uint64_t la = __shfl_sync(same, a, leader), lb = __shfl_sync(same, b, leader);
    const int32_t lc = __shfl_sync(same, c, leader);
    if (la != a || lb != b || lc != c) e = px_find_or_insert(t, a, b, c, &nw);      // folded keys collided: probe for myself
    *is_new = nw;
    return e;
}

__device__ __forceinline__ int32_t warp_min(int32_t v) { return __reduce_min_sync(0xffffffffu, v); }
__device__ __forceinline__ long long warp_max64(long long v) {
    for (int o = 16; o > 0; o >>= 1) { const long long w = __shfl_xor_sync(0xffffffffu, v, o); v = w > v ? w : v; }
    return v;
}

// ------------------------------------------------------------------ coordinator rule kernels
__global__ void k_px_rule_begin(PxScal* sc) {
    sc->max_rank = LLONG_MIN; sc->first_nonempty = INT_MAX; sc->first_collected = INT_MAX; sc->n_collected = 0;
    sc->distinct = 0; sc->kth_min = INT_MAX; sc->chosen = -1; sc->overflow = 0;
}

// max vrnd (:272-274) and the first message with a non-empty vval (:318-322)
__global__ void k_px_rule_max(int64_t m, const int64_t* __restrict__ vr, const int32_t* __restrict__ len, PxScal* __restrict__ sc) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    long long r = LLONG_MIN;
    int32_t fn = INT_MAX;
    if (i < m) { r = vr[i]; if (len[i] > 0) fn = (int32_t)i; }
    r = warp_max64(r);
    fn = warp_min(fn);
    if ((threadIdx.x & 31) == 0) {
        atomicMax(&sc->max_rank, r);
        if (fn != INT_MAX) atomicMin(&sc->first_nonempty, fn);
    }
}

// collectedVvals (:278-282): key[i] = table slot of the value of a collected message, T otherwise
__global__ void k_px_rule_collect(int64_t m, const int64_t* __restrict__ vr, const uint64_t* __restrict__ h1,
                                  const uint64_t* __restrict__ h2, const int32_t* __restrict__ len, PxTable t,
                                  uint32_t* __restrict__ key, int32_t* __restrict__ idx, PxScal* __restrict__ sc) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool col = false;
    int32_t fc = INT_MAX;
    const bool want = i < m && vr[i] == sc->max_rank && len[i] > 0;
    bool nw;
    const int32_t e = px_find_or_insert_warp(t, want, want ? h1[i] : 0, want ? h2[i] : 0, want ? len[i] : 0, &nw);
    if (i < m) {
        idx[i] = (int32_t)i;
        uint32_t k = t.T;
        if (want) {
            if (e < 0) atomicExch(&sc->overflow, 1);
            else {
                if (nw) atomicAdd(&sc->distinct, 1);
                k = (uint32_t)e; col = true; fc = (int32_t)i;
            }
        }
        key[i] = k;
    }
    const unsigned b = __ballot_sync(0xffffffffu, col);
    fc = warp_min(fc);
    if ((threadIdx.x & 31) == 0 && b) { atomicAdd(&sc->n_collected, __popc(b)); atomicMin(&sc->first_collected, fc); }
}

// the shared primitive: over keys sorted stably with their arrival indexes, find for every key the element at offset
// (need - 1 - prior[key]) of its run; the earliest such arrival index wins.  prior == NULL means 0 everywhere; if
// prior is given it is advanced by the run length (the per-round sender counts of the learner).
__global__ void k_px_kth(int64_t m, const uint32_t* __restrict__ skey, const int32_t* __restrict__ sval, uint32_t T,
                         const PxEntry* __restrict__ prior, int32_t need, int32_t* __restrict__ out_min) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    const uint32_t k = skey[p];
    if (k >= T) return;
    int64_t lo = 0, hi = p;                                  // first position of k's run (keys are sorted)
    while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (skey[mid] < k) lo = mid + 1; else hi = mid; }
    const int64_t off = p - lo;
    const int32_t before = prior ? prior[k].val : 0;             // read-only here; k_px_kth_advance updates it afterwards
    if (before < need && off == (int64_t)(need - 1 - before)) atomicMin(out_min, sval[p]);
}
__global__ void k_px_kth_advance(int64_t m, const uint32_t* __restrict__ skey, uint32_t T, PxEntry* __restrict__ prior) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    const uint32_t k = skey[p];
    if (k >= T) return;
    if (p + 1 < m && skey[p + 1] == k) return;               // only the last element of a run
    int64_t lo = 0, hi = p;
    while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (skey[mid] < k) lo = mid + 1; else hi = mid; }
    prior[k].val += (int32_t)(p - lo + 1);
}

// :287-326 — put the three cases together
__global__ void k_px_rule_final(const uint64_t* __restrict__ h1, const uint64_t* __restrict__ h2, const int32_t* __restrict__ len,
                                PxScal* __restrict__ sc) {
    int32_t c = -1;
    if (sc->distinct == 1) c = sc->first_collected;                                  // :287-289
    else if (sc->n_collected > 1 && sc->kth_min != INT_MAX) c = sc->kth_min;         // :293-308
    if (c < 0 && sc->first_nonempty != INT_MAX) c = sc->first_nonempty;              // :318-326
    sc->chosen = c;
    if (c >= 0) { sc->h1 = h1[c]; sc->h2 = h2[c]; sc->len = len[c]; } else { sc->h1 = 0; sc->h2 = 0; sc->len = 0; }
}

// ------------------------------------------------------------------ message staging kernels
__global__ void k_px_pack(int64_t n, const int32_t* __restrict__ round, const int32_t* __restrict__ node, int64_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = pack_rank(round[i], node[i]);
}
__global__ void k_px_table_clear(uint32_t T, PxEntry* __restrict__ e) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T) return;
    PxEntry z;
    z.state = 0; z.c = 0; z.a = 0; z.b = 0; z.val = INT_MAX; z.pad_ = 0;
    e[i] = z;
}

// phase1b filter (:160-167): keep[i] = cfg matches and rnd == crnd.   rnd == NULL: every message carries rnd_const.
__global__ void k_px1b_keep(int64_t n, const int64_t* __restrict__ mcfg, int64_t cfg, const int64_t* __restrict__ rnd,
                            int64_t rnd_const, int64_t crnd, int32_t* __restrict__ keep) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t r = rnd ? rnd[i] : rnd_const;
    keep[i] = (!(mcfg && mcfg[i] != cfg) && r == crnd) ? 1 : 0;
}
// append the kept messages to the coordinator's list in arrival order (:171)
__global__ void k_px1b_append(int64_t n, const int32_t* __restrict__ keep, const int32_t* __restrict__ pos, int64_t base,
                              const int64_t* __restrict__ vr, const uint64_t* __restrict__ h1, const uint64_t* __restrict__ h2,
                              const int32_t* __restrict__ len, int64_t* __restrict__ L_vr, uint64_t* __restrict__ L_h1,
                              uint64_t* __restrict__ L_h2, int32_t* __restrict__ L_len, int32_t* __restrict__ app_src,
                              PxScal* __restrict__ sc) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int32_t fn = INT_MAX;
    if (i < n) {
        if (keep[i]) {
            const int64_t j = base + pos[i];
            const int32_t l = len[i];
            L_vr[j] = vr[i]; L_h1[j] = h1[i]; L_h2[j] = h2 ? h2[i] : 0; L_len[j] = l;
            app_src[pos[i]] = (int32_t)i;
            if (l > 0) fn = pos[i];
        }
        if (i == n - 1) sc->kept = pos[i] + keep[i];
    }
    fn = warp_min(fn);
    if ((threadIdx.x & 31) == 0 && fn != INT_MAX) atomicMin(&sc->batch_first_nonempty, fn);
}
__global__ void k_px1b_begin(PxScal* sc) { sc->kept = 0; sc->batch_first_nonempty = INT_MAX; sc->src = -1; }
__global__ void k_px1b_src(const int32_t* __restrict__ app_src, int64_t at, PxScal* __restrict__ sc) { sc->src = app_src[at]; }

// ------------------------------------------------------------------ phase2b kernels
__global__ void k_px2b_begin(PxScal* sc) { sc->decide_idx = INT_MAX; sc->overflow = 0; sc->inserted = 0; }

// acceptResponses[rnd].put(sender, msg) (:228-230): slot of the (rnd, sender) pair; earliest arrival of a NEW pair wins it
__global__ void k_px2b_pairs(int64_t n, const int64_t* __restrict__ mcfg, int64_t cfg, const int64_t* __restrict__ rnd,
                             int64_t rnd_const, const int32_t* __restrict__ sender, PxTable t,
                             int32_t* __restrict__ slot, PxScal* __restrict__ sc) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int32_t e = -1;
    if (!(mcfg && mcfg[i] != cfg)) {
        bool nw;
        e = px_find_or_insert(t, (uint64_t)(rnd ? rnd[i] : rnd_const), (uint64_t)(uint32_t)sender[i], 0, &nw);
        if (e < 0) atomicExch(&sc->overflow, 1);
        else {
            if (nw) atomicAdd(&sc->inserted, 1);
            atomicMin(&t.e[e].val, (int32_t)i);            // INT_MAX on a fresh entry, -1 once a pair is from an earlier call
        }
    }
    slot[i] = e;
}
// key[i] = slot of the round's counter if message i is the first of its (rnd, sender) pair, T otherwise
__global__ void k_px2b_rounds(int64_t n, const int64_t* __restrict__ rnd, int64_t rnd_const, const int32_t* __restrict__ slot,
                              PxTable t, uint32_t* __restrict__ key, int32_t* __restrict__ idx,
                              PxScal* __restrict__ sc) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int32_t e = i < n ? slot[i] : -1;
    const bool first = e >= 0 && t.e[e].val == (int32_t)i;
    bool nw;
    const int32_t r = px_find_or_insert_warp(t, first, first ? (uint64_t)(rnd ? rnd[i] : rnd_const) : 0, 0, 1, &nw);   // c = 1: a round counter
    if (i >= n) return;
    idx[i] = (int32_t)i;
    uint32_t k = t.T;
    if (first) {
        if (r < 0) atomicExch(&sc->overflow, 1);
        else { if (nw) atomicAdd(&sc->inserted, 1); k = (uint32_t)r; }
    }
    key[i] = k;
}
// decoded Phase2b messages: the first one of the current configuration whose sender is outside the dictionary (-1)
__global__ void k_px2b_unknown(int64_t n, const int64_t* __restrict__ mcfg, int64_t cfg, const int32_t* __restrict__ sender,
                               PxScal* __restrict__ sc) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && mcfg[i] == cfg && sender[i] < 0) atomicMin(&sc->unknown_sender, (int32_t)i);
}
__global__ void k_px2b_unknown_begin(PxScal* sc) { sc->unknown_sender = INT_MAX; }
// the pairs of this call are "seen" from now on
__global__ void k_px2b_seal(int64_t n, const int32_t* __restrict__ slot, PxEntry* __restrict__ ent) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t e = slot[i];
    if (e >= 0 && ent[e].val == (int32_t)i) ent[e].val = -1;
}
__global__ void k_px2b_final(const uint64_t* __restrict__ h1, const uint64_t* __restrict__ h2, const int32_t* __restrict__ len,
                             uint64_t h1c, uint64_t h2c, int32_t lenc, PxScal* __restrict__ sc) {
    const int32_t d = sc->decide_idx;
    if (d != INT_MAX) {
        sc->h1 = h1 ? h1[d] : h1c; sc->h2 = h1 ? (h2 ? h2[d] : 0) : h2c; sc->len = h1 ? len[d] : lenc;
    }
}
// a round counter's prior count lives in the entry's val too (c == 1 entries); fresh entries hold INT_MAX -> 0
__global__ void k_px2b_fix_counters(int64_t m, const uint32_t* __restrict__ skey, uint32_t T, PxEntry* __restrict__ ent) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= m) return;
    const uint32_t k = skey[p];
    if (k >= T) return;
    if (p > 0 && skey[p - 1] == k) return;                   // first element of a run
    if (ent[k].val == INT_MAX) ent[k].val = 0;
}

// ------------------------------------------------------------------ acceptor kernels
__global__ void k_pxa_init(int64_t R, int64_t* rnd, int64_t* vrnd, uint64_t* h1, uint64_t* h2, int32_t* len) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    rnd[r] = pack_rank(0, 0); vrnd[r] = pack_rank(0, 0); h1[r] = 0; h2[r] = 0; len[r] = 0;     // Paxos.java:82-85
}
// A list of votes may name an acceptor more than once: win[r] (-1 before the call) becomes the last list index naming r.
__global__ void k_pxa_claim(int64_t n, const int64_t* __restrict__ acceptor, int64_t R, int32_t* __restrict__ win,
                            int32_t* __restrict__ bad) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t r = acceptor[i];
    if (r < 0 || r >= R) { atomicExch(bad, 1); return; }
    atomicMax(&win[r], (int32_t)i);
}
// registerFastRoundVote (:244-257).  acceptor == NULL: acceptor r takes vote r where flag[r] has RF_ANN_NOW.  With a list,
// only the entry k_pxa_claim left in win[r] writes acceptor r, so r ends with its last listed vote whole, as calls made one by
// one in list order would leave it; a list naming an acceptor out of range (*bad) writes nothing.
__global__ void k_pxa_register(int64_t n, const int64_t* __restrict__ acceptor, const int32_t* __restrict__ win,
                               const uint32_t* __restrict__ rflags, const uint64_t* __restrict__ vh1,
                               const uint64_t* __restrict__ vh2, const int32_t* __restrict__ vlen, int64_t* __restrict__ rnd,
                               int64_t* __restrict__ vrnd, uint64_t* __restrict__ h1, uint64_t* __restrict__ h2,
                               int32_t* __restrict__ len, const int32_t* __restrict__ bad) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int64_t r = i;
    if (acceptor) { if (*bad) return; r = acceptor[i]; if (win[r] != (int32_t)i) return; }
    else if (!(rflags[i] & RF_ANN_NOW)) return;
    if (rank_round(rnd[r]) > 1) return;                                              // :246-248
    rnd[r] = pack_rank(1, 1); vrnd[r] = pack_rank(1, 1);                             // :254-255
    h1[r] = vh1[i]; h2[r] = vh2 ? vh2[i] : 0; len[r] = vlen[i];                      // :256
}
// handlePhase1aMessage (:120-151) for one message; reply[r] = 1 where a Phase1bMessage goes back.  A silent acceptor (a
// crashed process, rapid_pxa_set_silent) neither changes nor answers.
__global__ void k_pxa_phase1a(int64_t R, int64_t rank, const uint8_t* __restrict__ silent, int64_t* __restrict__ rnd,
                              int32_t* __restrict__ reply) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    if (silent && silent[r]) { reply[r] = 0; return; }
    const bool up = rnd[r] < rank;                                                   // compareRanks(rnd, m.rank) < 0
    if (up) rnd[r] = rank;
    reply[r] = up ? 1 : 0;
}
// handlePhase2aMessage (:198-216) for one message; reply[r] = 1 where a Phase2bMessage is broadcast
__global__ void k_pxa_phase2a(int64_t R, int64_t mr, uint64_t vh1, uint64_t vh2, int32_t vlen, const uint8_t* __restrict__ silent,
                              int64_t* __restrict__ rnd, int64_t* __restrict__ vrnd, uint64_t* __restrict__ h1, uint64_t* __restrict__ h2,
                              int32_t* __restrict__ len, int32_t* __restrict__ reply) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    if (silent && silent[r]) { reply[r] = 0; return; }
    const bool acc = rnd[r] <= mr && vrnd[r] != mr;                                  // :204
    if (acc) { rnd[r] = mr; vrnd[r] = mr; h1[r] = vh1; h2[r] = vh2; len[r] = vlen; }
    reply[r] = acc ? 1 : 0;
}
// lowest acceptor holding vval == (vh1, vh2, vlen): per warp a shuffle min, then one atomicMin per warp (*out = R before)
__global__ void k_pxa_find(int64_t R, uint64_t vh1, uint64_t vh2, int32_t vlen, const uint64_t* __restrict__ h1,
                           const uint64_t* __restrict__ h2, const int32_t* __restrict__ len, unsigned long long* __restrict__ out) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long best = (unsigned long long)R;
    if (r < R && len[r] == vlen && h1[r] == vh1 && h2[r] == vh2) best = (unsigned long long)r;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
    if ((threadIdx.x & 31) == 0 && best < (unsigned long long)R) atomicMin(out, best);
}
// compact the answering acceptors (arrival order = acceptor order, or by permutation key)
__global__ void k_pxa_gather1b(int64_t R, const int32_t* __restrict__ reply, const int32_t* __restrict__ pos, int64_t begin,
                               const int64_t* __restrict__ vrnd, const uint64_t* __restrict__ h1, const uint64_t* __restrict__ h2,
                               const int32_t* __restrict__ len, int32_t* __restrict__ o_sender, int64_t* __restrict__ o_vr,
                               uint64_t* __restrict__ o_h1, uint64_t* __restrict__ o_h2, int32_t* __restrict__ o_len) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R || !reply[r]) return;
    const int32_t j = pos[r];
    o_sender[j] = (int32_t)(begin + r);
    if (o_vr) { o_vr[j] = vrnd[r]; o_h1[j] = h1[r]; o_h2[j] = h2[r]; o_len[j] = len[r]; }
}
__global__ void k_pxa_total(int64_t R, const int32_t* __restrict__ reply, const int32_t* __restrict__ pos, int32_t* __restrict__ out) {
    if (R > 0) *out = pos[R - 1] + reply[R - 1]; else *out = 0;
}
__global__ void k_px_perm_keys(int64_t n, const int32_t* __restrict__ sender, uint64_t seed, uint64_t* __restrict__ key, int32_t* __restrict__ idx) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    key[i] = splitmix64(seed ^ (uint64_t)(uint32_t)sender[i]);
    idx[i] = (int32_t)i;
}
template <typename T>
__global__ void k_px_gather(int64_t n, const int32_t* __restrict__ order, const T* __restrict__ in, T* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[order[i]];
}

// ------------------------------------------------------------------ handles
struct PxSeg;
struct PxRankHdr;
struct PX {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    float last_ms = 0.f;
    int64_t cfg = 0, N = 0, cap = 0;
    // coordinator (:67-71)
    int64_t crnd = pack_rank(0, 0);
    bool have_cval = false;
    uint64_t cval_h1 = 0, cval_h2 = 0;
    int32_t cval_len = 0;
    int64_t n_msgs = 0, first_nonempty = -1;
    DevBuf<int64_t> L_vr;
    DevBuf<uint64_t> L_h1, L_h2;
    DevBuf<int32_t> L_len;
    // learner (:68, :72)
    bool decided = false;
    uint64_t dec_h1 = 0, dec_h2 = 0;
    int32_t dec_len = 0;
    int64_t pairs = 0;                     // entries used in the persistent table
    uint32_t T = 0;                        // persistent (rnd, sender) / round-counter table
    DevBuf<PxEntry> tbl;
    // scratch
    uint32_t RT = 0;                       // rule table (cleared per evaluation)
    DevBuf<PxEntry> rtbl;
    DevBuf<uint32_t> key, skey;
    DevBuf<int32_t> idx, sidx, keep, pos, app_src, slot, scan_sums;
    RadixScratch rs;
    DevBuf<PxScal> sc;
    PinnedBuf<PxScal> h_sc;
    // staging of host message arrays (px_stage), and the packed ranks of every message batch
    DevBuf<int64_t> s_cfg, s_rnd, s_vr;
    DevBuf<int32_t> s_rnd_round, s_rnd_node, s_vrnd_round, s_vrnd_node, s_len, s_sender;
    DevBuf<uint64_t> s_h1, s_h2;
    // permuted deliveries
    DevBuf<uint64_t> pkey, spkey, g_h1, g_h2;
    DevBuf<int64_t> g_vr;
    DevBuf<int32_t> g_len, g_sender;
    // answers gathered from acceptor shards (ascending sender), and the exchange that brings them
    DevBuf<int32_t> sh_sender, sh_len;
    DevBuf<int64_t> sh_vr;
    DevBuf<uint64_t> sh_h1, sh_h2;
    DevBuf<unsigned char> stage, recv;     // this rank's packed answers / every rank's
    DevBuf<PxSeg> seg;
    PinnedBuf<PxSeg> h_seg;
    DevBuf<PxRankHdr> d_hdr;
    PinnedBuf<PxRankHdr> h_hdr;
    DevBuf<int32_t> d_ok;
    PinnedBuf<int32_t> h_ok;
};

struct PXA {
    int device = 0;
    cudaStream_t stream = nullptr;
    int64_t cfg = 0, R = 0, begin = 0;
    DevBuf<int64_t> rnd, vrnd;
    DevBuf<uint64_t> h1, h2;
    DevBuf<int32_t> len;
    // answers of the last phase1a / phase2a
    int last_kind = 0;                     // 0 none, 1 Phase1b answers, 2 Phase2b broadcasts
    int64_t last_rank = 0, n_out = 0;
    uint64_t last_h1 = 0, last_h2 = 0;
    int32_t last_len = 0;
    DevBuf<int32_t> reply, pos, o_sender, o_len, total;
    DevBuf<int64_t> o_vr;
    DevBuf<uint64_t> o_h1, o_h2;
    DevBuf<int32_t> scan_sums;
    PinnedBuf<int32_t> h_total;
    DevBuf<int32_t> bad, win;              // win: last list entry per acceptor of a vote registration
    DevBuf<int64_t> s_acc;
    DevBuf<uint64_t> s_h1, s_h2;
    DevBuf<int32_t> s_len;
    DevBuf<uint8_t> silent;                // crashed acceptors (rapid_pxa_set_silent); has_silent == false: every acceptor answers
    bool has_silent = false;
    DevBuf<unsigned long long> found;
    PinnedBuf<unsigned long long> h_found;
};

static const int TB = 256;
static inline unsigned grid_for(int64_t n) { return (unsigned)ceil_div<int64_t>(n > 0 ? n : 1, TB); }

static int32_t px_scratch(PX* px, int64_t n) {
    RAPID_CHECK(px->key.reserve((size_t)n)); RAPID_CHECK(px->skey.reserve((size_t)n));
    RAPID_CHECK(px->idx.reserve((size_t)n)); RAPID_CHECK(px->sidx.reserve((size_t)n));
    RAPID_CHECK(px->keep.reserve((size_t)n)); RAPID_CHECK(px->pos.reserve((size_t)n));
    RAPID_CHECK(px->app_src.reserve((size_t)n)); RAPID_CHECK(px->slot.reserve((size_t)n));
    return RAPID_OK;
}

// stable sort of (key, idx) by the low `bits` bits of the key (radix.cuh, hand-written; inputs only read)
static int32_t px_sort_pairs(PX* px, int64_t m, int bits) {
    return radix_sort_pairs<uint32_t>(px->rs, px->key.p, px->idx.p, px->skey.p, px->sidx.p, m, 0, bits, px->stream, false);
}
static int bits_for(uint32_t T) { int b = 1; while ((1ull << b) <= (uint64_t)T) ++b; return b; }   // keys in [0, T]

// selectProposalUsingCoordinatorRule over device arrays; leaves chosen / value in px->sc (no readback here)
static int32_t px_rule_device(PX* px, int64_t m, const int64_t* vr, const uint64_t* h1, const uint64_t* h2, const int32_t* len) {
    cudaStream_t s = px->stream;
    uint32_t RT = 1024;
    while ((int64_t)RT < 2 * m) RT <<= 1;
    if (RT > px->RT) {
        RAPID_CHECK(px->rtbl.reserve(RT));
        px->RT = RT;
    }
    RT = px->RT;
    RAPID_CHECK(px_scratch(px, m));
    k_px_table_clear<<<grid_for(RT), TB, 0, s>>>(RT, px->rtbl.p);
    PxTable t{RT, px->rtbl.p};
    k_px_rule_begin<<<1, 1, 0, s>>>(px->sc.p);
    k_px_rule_max<<<grid_for(m), TB, 0, s>>>(m, vr, len, px->sc.p);
    k_px_rule_collect<<<grid_for(m), TB, 0, s>>>(m, vr, h1, h2, len, t, px->key.p, px->idx.p, px->sc.p);
    RAPID_KERNEL_CHECK();
    RAPID_CHECK(px_sort_pairs(px, m, bits_for(RT)));
    k_px_kth<<<grid_for(m), TB, 0, s>>>(m, px->skey.p, px->sidx.p, RT, nullptr, (int32_t)(px->N / 4) + 1, &px->sc.p->kth_min);
    k_px_rule_final<<<1, 1, 0, s>>>(h1, h2, len, px->sc.p);
    RAPID_KERNEL_CHECK();
    return RAPID_OK;
}

static int32_t px_read_scal(PX* px) {
    RAPID_CUDA(cudaMemcpyAsync(px->h_sc.p, px->sc.p, sizeof(PxScal), cudaMemcpyDeviceToHost, px->stream));
    RAPID_CUDA(cudaStreamSynchronize(px->stream));
    return RAPID_OK;
}

// Runs `body` on the px's device between ev0 and ev1.  Only a call that succeeds waits for ev1 and sets what
// rapid_px_last_device_ms reports.
template <class F>
static int32_t px_timed(PX* px, F&& body) {
    DeviceGuard g(px->device);
    RAPID_CUDA(cudaEventRecord(px->ev0, px->stream));
    const int32_t rc = body();
    if (rc == RAPID_OK) { cudaEventRecord(px->ev1, px->stream); cudaEventSynchronize(px->ev1); cudaEventElapsedTime(&px->last_ms, px->ev0, px->ev1); }
    return rc;
}

// handlePhase1bMessage over device arrays (rnd == NULL: every message carries rnd_const; mcfg == NULL: cfg)
static int32_t px_phase1b_device(PX* px, int64_t n, const int64_t* mcfg, const int64_t* rnd, int64_t rnd_const, const int64_t* vr,
                                 const uint64_t* h1, const uint64_t* h2, const int32_t* len, int32_t* proposed,
                                 int64_t* trigger_index, uint64_t* ch1, uint64_t* ch2, int32_t* clen, int64_t* n_messages) {
    cudaStream_t s = px->stream;
    if (proposed) *proposed = 0;
    if (trigger_index) *trigger_index = -1;
    if (n > 0) {
        {   // the list grows past message_capacity if it must (a batch may be mostly filtered; the bound is only known afterwards)
            const size_t need = (size_t)(px->n_msgs + n);
            RAPID_CHECK(px->L_vr.reserve(need, true, s)); RAPID_CHECK(px->L_h1.reserve(need, true, s));
            RAPID_CHECK(px->L_h2.reserve(need, true, s)); RAPID_CHECK(px->L_len.reserve(need, true, s));
        }
        RAPID_CHECK(px_scratch(px, n));
        k_px1b_begin<<<1, 1, 0, s>>>(px->sc.p);
        k_px1b_keep<<<grid_for(n), TB, 0, s>>>(n, mcfg, px->cfg, rnd, rnd_const, px->crnd, px->keep.p);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(exclusive_scan_i32_to(px->keep.p, px->pos.p, n, px->scan_sums, s));
        k_px1b_append<<<grid_for(n), TB, 0, s>>>(n, px->keep.p, px->pos.p, px->n_msgs, vr, h1, h2, len, px->L_vr.p, px->L_h1.p,
                                                  px->L_h2.p, px->L_len.p, px->app_src.p, px->sc.p);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(px_read_scal(px));
        const int64_t old = px->n_msgs, total = old + px->h_sc.p->kept;
        if (px->first_nonempty < 0 && px->h_sc.p->batch_first_nonempty != INT_MAX) px->first_nonempty = old + px->h_sc.p->batch_first_nonempty;
        px->n_msgs = total;
        if (!px->have_cval && px->first_nonempty >= 0) {
            // size() > N/2 (:173) <=> arrival index >= N/2; the rule's result is non-empty from the first non-empty vval on
            int64_t jstar = px->N / 2;
            if (px->first_nonempty > jstar) jstar = px->first_nonempty;
            if (old > jstar) jstar = old;                     // the rule only runs when a message arrives
            if (jstar < total) {
                k_px1b_src<<<1, 1, 0, s>>>(px->app_src.p, jstar - old, px->sc.p);     // before the rule regrows the scratch
                RAPID_KERNEL_CHECK();
                RAPID_CHECK(px_rule_device(px, jstar + 1, px->L_vr.p, px->L_h1.p, px->L_h2.p, px->L_len.p));
                RAPID_CHECK(px_read_scal(px));
                const PxScal& r = *px->h_sc.p;
                if (r.overflow) { set_error("internal: rule table overflow"); return RAPID_ECUDA; }
                if (r.chosen < 0 || r.len <= 0) { set_error("internal: coordinator rule returned an empty value"); return RAPID_ECUDA; }
                px->have_cval = true; px->cval_h1 = r.h1; px->cval_h2 = r.h2; px->cval_len = r.len;      // :181
                if (proposed) *proposed = 1;
                if (trigger_index) *trigger_index = r.src;
            }
        }
    }
    if (ch1) *ch1 = px->have_cval ? px->cval_h1 : 0;
    if (ch2) *ch2 = px->have_cval ? px->cval_h2 : 0;
    if (clen) *clen = px->have_cval ? px->cval_len : 0;
    if (n_messages) *n_messages = px->n_msgs;
    return RAPID_OK;
}

// handlePhase2bMessage over device arrays (h1 == NULL: every message carries (h1c, h2c, lenc))
static int32_t px_phase2b_device(PX* px, int64_t n, const int64_t* mcfg, const int64_t* rnd, int64_t rnd_const, const int32_t* sender,
                                 const uint64_t* h1, const uint64_t* h2, const int32_t* len, uint64_t h1c, uint64_t h2c, int32_t lenc,
                                 int32_t* decided, int64_t* decided_index, uint64_t* dh1, uint64_t* dh2, int32_t* dlen) {
    cudaStream_t s = px->stream;
    if (decided_index) *decided_index = -1;
    if (n > 0) {
        // worst case this call adds n new (rnd, sender) pairs and n new rounds: refuse before the table degrades
        if (px->pairs + 2 * n > (int64_t)px->T / 4 * 3) { set_error("Phase2b table would exceed message_capacity (%lld)", (long long)px->cap); return RAPID_ENOMEM; }
        RAPID_CHECK(px_scratch(px, n));
        PxTable t{px->T, px->tbl.p};
        k_px2b_begin<<<1, 1, 0, s>>>(px->sc.p);
        k_px2b_pairs<<<grid_for(n), TB, 0, s>>>(n, mcfg, px->cfg, rnd, rnd_const, sender, t, px->slot.p, px->sc.p);
        k_px2b_rounds<<<grid_for(n), TB, 0, s>>>(n, rnd, rnd_const, px->slot.p, t, px->key.p, px->idx.p, px->sc.p);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(px_sort_pairs(px, n, bits_for(px->T)));
        k_px2b_fix_counters<<<grid_for(n), TB, 0, s>>>(n, px->skey.p, px->T, px->tbl.p);
        k_px_kth<<<grid_for(n), TB, 0, s>>>(n, px->skey.p, px->sidx.p, px->T, px->tbl.p, (int32_t)(px->N / 2) + 1, &px->sc.p->decide_idx);
        k_px_kth_advance<<<grid_for(n), TB, 0, s>>>(n, px->skey.p, px->T, px->tbl.p);
        k_px2b_seal<<<grid_for(n), TB, 0, s>>>(n, px->slot.p, px->tbl.p);
        k_px2b_final<<<1, 1, 0, s>>>(h1, h2, len, h1c, h2c, lenc, px->sc.p);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(px_read_scal(px));
        const PxScal& r = *px->h_sc.p;
        if (r.overflow) { set_error("Phase2b table full (message_capacity too small)"); return RAPID_ENOMEM; }
        px->pairs += r.inserted;
        if (!px->decided && r.decide_idx != INT_MAX) {                               // :231-235
            px->decided = true; px->dec_h1 = r.h1; px->dec_h2 = r.h2; px->dec_len = r.len;
            if (decided_index) *decided_index = r.decide_idx;
        }
    }
    if (decided) *decided = px->decided ? 1 : 0;
    if (dh1) *dh1 = px->decided ? px->dec_h1 : 0;
    if (dh2) *dh2 = px->decided ? px->dec_h2 : 0;
    if (dlen) *dlen = px->decided ? px->dec_len : 0;
    return RAPID_OK;
}

// handlePhase1bMessage / handlePhase2bMessage over a batch of messages on the device, decoded from the wire or staged from host
// arrays: the ranks are packed, then tallied
static int32_t px_phase1b_msgs(PX* px, const WireMsgs& m, int32_t* proposed, int64_t* trigger_index, uint64_t* ch1, uint64_t* ch2,
                               int32_t* clen, int64_t* n_messages) {
    cudaStream_t s = px->stream;
    if (m.n > 0) {
        RAPID_CHECK(px->s_rnd.reserve((size_t)m.n)); RAPID_CHECK(px->s_vr.reserve((size_t)m.n));
        k_px_pack<<<grid_for(m.n), TB, 0, s>>>(m.n, m.rnd_round, m.rnd_node, px->s_rnd.p);
        k_px_pack<<<grid_for(m.n), TB, 0, s>>>(m.n, m.vrnd_round, m.vrnd_node, px->s_vr.p);
        RAPID_KERNEL_CHECK();
    }
    return px_phase1b_device(px, m.n, m.cfg, px->s_rnd.p, 0, px->s_vr.p, m.h1, m.h2, m.len, proposed, trigger_index, ch1, ch2, clen,
                             n_messages);
}
static int32_t px_phase2b_msgs(PX* px, const WireMsgs& m, int32_t* decided, int64_t* decided_index, uint64_t* dh1, uint64_t* dh2,
                               int32_t* dlen) {
    if (m.n > 0) {
        RAPID_CHECK(px->s_rnd.reserve((size_t)m.n));
        k_px_pack<<<grid_for(m.n), TB, 0, px->stream>>>(m.n, m.rnd_round, m.rnd_node, px->s_rnd.p);
        RAPID_KERNEL_CHECK();
    }
    return px_phase2b_device(px, m.n, m.cfg, px->s_rnd.p, 0, m.sender, m.h1, m.h2, m.len, 0, 0, 0, decided, decided_index, dh1, dh2,
                             dlen);
}

template <typename T>
static int32_t upload(DevBuf<T>& d, const T* h, int64_t n, cudaStream_t s) {
    RAPID_CHECK(d.reserve((size_t)(n > 0 ? n : 1)));
    if (n > 0) RAPID_CUDA(cudaMemcpyAsync(d.p, h, (size_t)n * sizeof(T), cudaMemcpyHostToDevice, s));
    return RAPID_OK;
}

// n messages of host arrays uploaded into the px's staging buffers, as a WireMsgs; an array passed as NULL stays NULL
template <typename T>
static int32_t stage(DevBuf<T>& d, const T* h, int64_t n, cudaStream_t s, const T** out) {
    *out = nullptr;
    if (h) { RAPID_CHECK(upload(d, h, n, s)); *out = d.p; }
    return RAPID_OK;
}
static int32_t px_stage(PX* px, int64_t n, const int64_t* cfg, const int32_t* rnd_round, const int32_t* rnd_node,
                        const int32_t* vrnd_round, const int32_t* vrnd_node, const int32_t* sender, const uint64_t* h1,
                        const uint64_t* h2, const int32_t* len, WireMsgs* m) {
    *m = WireMsgs{};
    m->device = px->device; m->n = n;
    if (n == 0) return RAPID_OK;
    cudaStream_t s = px->stream;
    RAPID_CHECK(stage(px->s_cfg, cfg, n, s, &m->cfg));
    RAPID_CHECK(stage(px->s_rnd_round, rnd_round, n, s, &m->rnd_round)); RAPID_CHECK(stage(px->s_rnd_node, rnd_node, n, s, &m->rnd_node));
    RAPID_CHECK(stage(px->s_vrnd_round, vrnd_round, n, s, &m->vrnd_round));
    RAPID_CHECK(stage(px->s_vrnd_node, vrnd_node, n, s, &m->vrnd_node));
    RAPID_CHECK(stage(px->s_sender, sender, n, s, &m->sender));
    RAPID_CHECK(stage(px->s_h1, h1, n, s, &m->h1)); RAPID_CHECK(stage(px->s_h2, h2, n, s, &m->h2));
    RAPID_CHECK(stage(px->s_len, len, n, s, &m->len));
    return RAPID_OK;
}

static int32_t check_device(int32_t device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); set_error("no CUDA device: librapid_b200 has no CPU fallback"); return RAPID_ECUDA; }
    if (device < 0 || device >= ndev) { set_error("device out of range"); return RAPID_EINVAL; }
    return RAPID_OK;
}

// arrival order of n compacted answers (sender ascending): order[i] = answer position delivered i-th (NULL = as compacted);
// with an order, px->g_sender holds the senders in arrival order
static int32_t px_arrival_order(PX* px, const int32_t* sender, int64_t n, uint64_t perm_seed, const int32_t** order) {
    *order = nullptr;
    if (perm_seed == 0 || n <= 1) return RAPID_OK;
    cudaStream_t s = px->stream;
    RAPID_CHECK(px->pkey.reserve((size_t)n)); RAPID_CHECK(px->spkey.reserve((size_t)n));
    RAPID_CHECK(px->idx.reserve((size_t)n)); RAPID_CHECK(px->sidx.reserve((size_t)n));
    k_px_perm_keys<<<grid_for(n), TB, 0, s>>>(n, sender, perm_seed, px->pkey.p, px->idx.p);
    RAPID_KERNEL_CHECK();
    RAPID_CHECK(radix_sort_pairs<uint64_t>(px->rs, px->pkey.p, px->idx.p, px->spkey.p, px->sidx.p, n, 0, 64, s, false));
    RAPID_CHECK(px->g_sender.reserve((size_t)n));
    k_px_gather<int32_t><<<grid_for(n), TB, 0, s>>>(n, px->sidx.p, sender, px->g_sender.p);
    RAPID_KERNEL_CHECK();
    *order = px->sidx.p;      // NOTE: valid until the next sort on this handle; callers gather before tallying
    return RAPID_OK;
}

// ------------------------------------------------------------------ answers of several acceptor shards
// Every shard (on every rank) contributes one fixed header; the gathered table is validated identically everywhere before any
// answer moves, then the compacted answers are packed, all-gathered and unpacked in ascending acceptor_begin, which for
// disjoint shards is exactly the compaction order (ascending sender) of one handle over their union.
static const int PX_MAX_SHARDS = 64;        // per rank: the header exchange has a fixed size

struct PxShardHdr {
    int64_t begin, R, n_out, last_rank, cfg;
    uint64_t h1, h2;                        // the Phase2a value (Phase2b answers only)
    int32_t len, kind, on_px_device, pad_;
};
struct PxRankHdr {
    int32_t n_shards, bad, want, pad_;      // bad: NULL shard or n_shards outside [1, PX_MAX_SHARDS]; want: 1 Phase1b, 2 Phase2b
    PxShardHdr s[PX_MAX_SHARDS];
};
struct __align__(16) Px1bRec {              // one Phase1b answer in the exchange: 32 B
    int32_t sender, len;
    int64_t vr;
    uint64_t h1, h2;
};
struct PxSeg { int64_t dst, src, n; };     // answers [dst, dst + n) of the gathered arrays come from records [src, src + n)

__global__ void k_px_pack1b(int64_t n, const int32_t* __restrict__ sender, const int64_t* __restrict__ vr, const uint64_t* __restrict__ h1,
                            const uint64_t* __restrict__ h2, const int32_t* __restrict__ len, Px1bRec* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Px1bRec r;
    r.sender = sender[i]; r.len = len[i]; r.vr = vr[i]; r.h1 = h1[i]; r.h2 = h2[i];
    out[i] = r;
}
__device__ __forceinline__ int32_t px_seg_of(const PxSeg* __restrict__ seg, int32_t nseg, int64_t j) {
    int32_t lo = 0, hi = nseg - 1;                           // last segment with dst <= j (segments are non-empty and ascending)
    while (lo < hi) { const int32_t mid = (lo + hi + 1) >> 1; if (seg[mid].dst <= j) lo = mid; else hi = mid - 1; }
    return lo;
}
__global__ void k_px_unpack1b(int64_t n, const PxSeg* __restrict__ seg, int32_t nseg, const Px1bRec* __restrict__ in,
                              int32_t* __restrict__ sender, int64_t* __restrict__ vr, uint64_t* __restrict__ h1,
                              uint64_t* __restrict__ h2, int32_t* __restrict__ len) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const PxSeg g = seg[px_seg_of(seg, nseg, j)];
    const Px1bRec r = in[g.src + (j - g.dst)];
    sender[j] = r.sender; vr[j] = r.vr; h1[j] = r.h1; h2[j] = r.h2; len[j] = r.len;
}
__global__ void k_px_unpack2b(int64_t n, const PxSeg* __restrict__ seg, int32_t nseg, const int32_t* __restrict__ in,
                              int32_t* __restrict__ sender) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const PxSeg g = seg[px_seg_of(seg, nseg, j)];
    sender[j] = in[g.src + (j - g.dst)];
}

static int32_t px_clear_tables(PX* px) {
    k_px_table_clear<<<grid_for(px->T), TB, 0, px->stream>>>(px->T, px->tbl.p);
    RAPID_KERNEL_CHECK();
    return RAPID_OK;
}

}  // namespace rapid

using namespace rapid;

struct rapid_px : rapid::PX {};
struct rapid_pxa : rapid::PXA {};

void rapid::pxa_answers_dev(const rapid_pxa* a, PxaAnswers* out) {
    out->device = a->device; out->kind = a->last_kind; out->cfg = a->cfg; out->R = a->R; out->begin = a->begin;
    out->n = a->n_out; out->rank = a->last_rank;
    out->sender = a->o_sender.p; out->vrnd = a->o_vr.p; out->h1 = a->o_h1.p; out->h2 = a->o_h2.p; out->len = a->o_len.p;
    out->v_h1 = a->last_h1; out->v_h2 = a->last_h2; out->v_len = a->last_len;
}

// Gather the pending answers of `want` kind (1 Phase1b, 2 Phase2b) of this rank's shards and, with a comm, of every rank's into
// px->sh_* in ascending sender.  Every refusal that depends on the shards is decided from the gathered header table, which is
// the same on every rank, so either every rank returns it or every rank goes on to the data exchange.  One shard without a comm
// is already in that order and is read in place.  *out: the answers as one handle would hold them (R and begin left 0 for
// gathered ones), with the rank of the broadcast they answer and (Phase2b) its value.
static int32_t px_gather_shards(rapid_px* px, const rapid_pxa* const* shards, int32_t n_shards, rapid_comm* comm, int want,
                                PxaAnswers* out) {
    cudaStream_t s = px->stream;
    const int world = comm ? comm->world : 1, me = comm ? comm->rank : 0;
    if (comm && !g_nccl.AllGather) { set_error("libnccl lacks ncclAllGather"); return RAPID_ENCCL; }
    // 1. headers
    RAPID_CHECK(px->h_hdr.reserve((size_t)world));
    PxRankHdr& mine = px->h_hdr.p[me];
    memset(&mine, 0, sizeof(mine));
    mine.want = want;
    if (!shards || n_shards < 1 || n_shards > PX_MAX_SHARDS) mine.bad = 1;
    else {
        mine.n_shards = n_shards;
        for (int32_t i = 0; i < n_shards; ++i) {
            const rapid_pxa* a = shards[i];
            if (!a) { mine.bad = 1; break; }
            PxShardHdr& h = mine.s[i];
            h.begin = a->begin; h.R = a->R; h.n_out = a->n_out; h.last_rank = a->last_rank; h.cfg = a->cfg;
            h.kind = a->last_kind; h.on_px_device = a->device == px->device ? 1 : 0;
            if (a->last_kind == 2) { h.h1 = a->last_h1; h.h2 = a->last_h2; h.len = a->last_len; }
        }
    }
    if (comm) {
        RAPID_CHECK(px->d_hdr.reserve((size_t)world)); RAPID_CHECK(px->d_ok.reserve(1)); RAPID_CHECK(px->h_ok.reserve(1));
        RAPID_CUDA(cudaMemcpyAsync(px->d_hdr.p + me, &mine, sizeof(PxRankHdr), cudaMemcpyHostToDevice, s));
        RAPID_NCCL(g_nccl.AllGather(px->d_hdr.p + me, px->d_hdr.p, sizeof(PxRankHdr), NCCL_UINT8, comm->comm, s));
        RAPID_CUDA(cudaMemcpyAsync(px->h_hdr.p, px->d_hdr.p, (size_t)world * sizeof(PxRankHdr), cudaMemcpyDeviceToHost, s));
        RAPID_CUDA(cudaStreamSynchronize(s));
    }
    // 2. validate the gathered table (identical on every rank) and place every shard's answers
    struct Ent { int64_t begin, R, n_out, src; int r; };
    std::vector<Ent> all;
    std::vector<int64_t> rank_total((size_t)world, 0);
    const PxShardHdr* ref = nullptr;
    for (int r = 0; r < world; ++r) {
        const PxRankHdr& h = px->h_hdr.p[r];
        if (h.bad) { set_error("rank %d passed a NULL shard or n_shards outside [1, %d]", r, PX_MAX_SHARDS); return RAPID_EINVAL; }
        if (h.want != want) { set_error("ranks disagree on the tally: rank %d asked for Phase%db answers", r, h.want); return RAPID_EINVAL; }
        for (int32_t i = 0; i < h.n_shards; ++i) {
            const PxShardHdr& x = h.s[i];
            if (!x.on_px_device) { set_error("shard %d of rank %d lives on a device other than the px's", i, r); return RAPID_EINVAL; }
            if (x.kind != want) {
                if (want == 1) set_error("no Phase1b answers pending on shard %d of rank %d (call rapid_pxa_phase1a first)", i, r);
                else set_error("no Phase2b broadcasts pending on shard %d of rank %d (call rapid_pxa_phase2a first)", i, r);
                return RAPID_EINVAL;
            }
            if (!ref) ref = &x;
            else if (x.last_rank != ref->last_rank || x.cfg != ref->cfg || x.h1 != ref->h1 || x.h2 != ref->h2 || x.len != ref->len) {
                set_error("shard %d of rank %d answered a different broadcast (rank, configuration or Phase2a value)", i, r);
                return RAPID_EINVAL;
            }
            all.push_back({x.begin, x.R, x.n_out, rank_total[(size_t)r], r});
            rank_total[(size_t)r] += x.n_out;
        }
    }
    std::sort(all.begin(), all.end(), [](const Ent& a, const Ent& b) { return a.begin < b.begin; });
    for (size_t k = 1; k < all.size(); ++k)
        if (all[k - 1].begin + all[k - 1].R > all[k].begin) {
            set_error("acceptor ranges overlap: [%lld, %lld) and [%lld, %lld)", (long long)all[k - 1].begin,
                      (long long)(all[k - 1].begin + all[k - 1].R), (long long)all[k].begin, (long long)(all[k].begin + all[k].R));
            return RAPID_EINVAL;
        }
    if (!comm && n_shards == 1) {
        pxa_answers_dev(shards[0], out);
        return RAPID_OK;
    }
    const int64_t per_rank = *std::max_element(rank_total.begin(), rank_total.end());   // padded block of every rank
    int64_t n = 0;
    for (const Ent& e : all) n += e.n_out;
    const size_t rec = want == 1 ? sizeof(Px1bRec) : sizeof(int32_t);
    // 3. scratch for the gathered sizes; with a comm every rank learns whether every rank has it before the data moves
    const size_t nn = (size_t)std::max<int64_t>(n, 1), nseg = std::max<size_t>(all.size(), 1);
    const size_t block = (size_t)std::max<int64_t>(per_rank, 1) * rec;
    int32_t rc = px->stage.reserve(block);
    if (!rc && comm) rc = px->recv.reserve((size_t)world * block);
    if (!rc) rc = px->sh_sender.reserve(nn);
    if (!rc && want == 1) rc = px->sh_vr.reserve(nn);
    if (!rc && want == 1) rc = px->sh_h1.reserve(nn);
    if (!rc && want == 1) rc = px->sh_h2.reserve(nn);
    if (!rc && want == 1) rc = px->sh_len.reserve(nn);
    if (!rc) rc = px->seg.reserve(nseg);
    if (!rc) rc = px->h_seg.reserve(nseg);
    if (comm) {
        *px->h_ok.p = rc == RAPID_OK ? 1 : 0;
        RAPID_CUDA(cudaMemcpyAsync(px->d_ok.p, px->h_ok.p, sizeof(int32_t), cudaMemcpyHostToDevice, s));
        RAPID_NCCL(g_nccl.AllReduce(px->d_ok.p, px->d_ok.p, 1, NCCL_INT32, NCCL_MIN, comm->comm, s));
        RAPID_CUDA(cudaMemcpyAsync(px->h_ok.p, px->d_ok.p, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
        RAPID_CUDA(cudaStreamSynchronize(s));
        if (rc == RAPID_OK && !*px->h_ok.p) { set_error("another rank could not allocate the exchange buffers"); return RAPID_ENOMEM; }
    }
    RAPID_CHECK(rc);
    // 4. pack this rank's answers (list order), exchange, unpack in ascending acceptor_begin
    int64_t off = 0;
    for (int32_t i = 0; i < n_shards; ++i) {
        const rapid_pxa* a = shards[i];
        const int64_t m = a->n_out;
        if (m > 0 && want == 1) {
            k_px_pack1b<<<grid_for(m), TB, 0, s>>>(m, a->o_sender.p, a->o_vr.p, a->o_h1.p, a->o_h2.p, a->o_len.p, (Px1bRec*)px->stage.p + off);
            RAPID_KERNEL_CHECK();
        } else if (m > 0) {                                  // Phase2b: the sender is the whole answer
            RAPID_CUDA(cudaMemcpyAsync((int32_t*)px->stage.p + off, a->o_sender.p, (size_t)m * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
        }
        off += m;
    }
    const unsigned char* in = px->stage.p;
    if (comm && per_rank > 0) {
        RAPID_NCCL(g_nccl.AllGather(px->stage.p, px->recv.p, (size_t)per_rank * rec, NCCL_UINT8, comm->comm, s));
        in = px->recv.p;
    }
    int32_t k = 0;
    int64_t dst = 0;
    for (const Ent& e : all) {
        if (e.n_out == 0) continue;
        px->h_seg.p[k++] = PxSeg{dst, (comm ? (int64_t)e.r * per_rank : 0) + e.src, e.n_out};
        dst += e.n_out;
    }
    if (n > 0) {
        RAPID_CUDA(cudaMemcpyAsync(px->seg.p, px->h_seg.p, (size_t)k * sizeof(PxSeg), cudaMemcpyHostToDevice, s));
        if (want == 1)
            k_px_unpack1b<<<grid_for(n), TB, 0, s>>>(n, px->seg.p, k, (const Px1bRec*)in, px->sh_sender.p, px->sh_vr.p, px->sh_h1.p,
                                                      px->sh_h2.p, px->sh_len.p);
        else
            k_px_unpack2b<<<grid_for(n), TB, 0, s>>>(n, px->seg.p, k, (const int32_t*)in, px->sh_sender.p);
        RAPID_KERNEL_CHECK();
    }
    *out = PxaAnswers{};
    out->device = px->device; out->kind = want; out->cfg = ref->cfg; out->n = n; out->rank = ref->last_rank;
    out->sender = px->sh_sender.p; out->vrnd = px->sh_vr.p; out->h1 = px->sh_h1.p; out->h2 = px->sh_h2.p; out->len = px->sh_len.p;
    out->v_h1 = ref->h1; out->v_h2 = ref->h2; out->v_len = ref->len;
    return RAPID_OK;
}

extern "C" {

int32_t rapid_px_create(rapid_px** out, int64_t cfg_id, int64_t membership_size, int64_t message_capacity, int32_t device) {
    if (!out || membership_size < 1 || message_capacity < 1 || message_capacity > 0x3ffffff0LL) { set_error("bad arguments"); return RAPID_EINVAL; }
    *out = nullptr;
    RAPID_CHECK(check_device(device));
    DeviceGuard g(device);
    rapid_px* px = new rapid_px();
    px->device = device; px->cfg = cfg_id; px->N = membership_size; px->cap = message_capacity;
    uint32_t T = 1024;
    while ((int64_t)T < 4 * message_capacity) T <<= 1;        // pairs + round counters, load <= 1/2
    px->T = T;
    int32_t rc = RAPID_OK;
    do {
        if (cudaStreamCreateWithFlags(&px->stream, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreate(&px->ev0) != cudaSuccess ||
            cudaEventCreate(&px->ev1) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "stream", __FILE__, __LINE__); break; }
        const size_t cap = (size_t)message_capacity;
        if ((rc = px->L_vr.reserve(cap)) || (rc = px->L_h1.reserve(cap)) || (rc = px->L_h2.reserve(cap)) || (rc = px->L_len.reserve(cap))) break;
        if ((rc = px->tbl.reserve(T))) break;
        if ((rc = px->sc.reserve(1)) || (rc = px->h_sc.reserve(1))) break;
        cudaMemsetAsync(px->sc.p, 0, sizeof(PxScal), px->stream);
        if ((rc = px_clear_tables(px))) break;
        if (cudaStreamSynchronize(px->stream) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "init", __FILE__, __LINE__); break; }
    } while (0);
    if (rc) { rapid_px_destroy(px); return rc; }
    *out = px;
    return RAPID_OK;
}

// The Paxos instance of the next configuration (FastPaxos ctor :86, MembershipService.java:427-429) on the same buffers.
int32_t rapid_px_reset(rapid_px* px, int64_t cfg_id, int64_t membership_size) {
    if (!px || membership_size < 1) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(px->device);
    px->cfg = cfg_id; px->N = membership_size;
    px->crnd = pack_rank(0, 0); px->have_cval = false; px->cval_h1 = px->cval_h2 = 0; px->cval_len = 0;
    px->n_msgs = 0; px->first_nonempty = -1;
    px->decided = false; px->dec_h1 = px->dec_h2 = 0; px->dec_len = 0; px->pairs = 0;
    return px_clear_tables(px);                               // asynchronous: ordered before the next call on the stream
}

int32_t rapid_px_destroy(rapid_px* px) {
    if (!px) return RAPID_OK;
    DeviceGuard g(px->device);
    if (px->stream) { cudaStreamSynchronize(px->stream); cudaStreamDestroy(px->stream); }
    if (px->ev0) cudaEventDestroy(px->ev0);
    if (px->ev1) cudaEventDestroy(px->ev1);
    delete px;
    return RAPID_OK;
}

int32_t rapid_px_start_phase1a(rapid_px* px, int32_t round, int32_t node_index, int32_t* started) {
    if (!px) { set_error("NULL handle"); return RAPID_EINVAL; }
    const bool go = !(rank_round(px->crnd) > round);          // :99-101
    if (go) px->crnd = pack_rank(round, node_index);          // :102
    if (started) *started = go ? 1 : 0;
    return RAPID_OK;
}

int32_t rapid_px_coordinator_rule(rapid_px* px, int64_t n, const int32_t* vrnd_round, const int32_t* vrnd_node, const uint64_t* vval_hash,
                                  const uint64_t* vval_hash2, const int32_t* vval_len, int64_t* chosen_index) {
    if (!px || !chosen_index) { set_error("NULL argument"); return RAPID_EINVAL; }
    if (n <= 0) { set_error("phase1bMessages was empty"); return RAPID_EINVAL; }                   // :274
    if (n > 0x7ffffff0LL || !vrnd_round || !vrnd_node || !vval_hash || !vval_len) { set_error("bad arguments"); return RAPID_EINVAL; }
    // timed apart from px_timed: ev1 is recorded before the readback, which goes out without waiting for it
    DeviceGuard g(px->device);
    cudaStream_t s = px->stream;
    RAPID_CUDA(cudaEventRecord(px->ev0, s));
    RAPID_CHECK(upload(px->s_vrnd_round, vrnd_round, n, s)); RAPID_CHECK(upload(px->s_vrnd_node, vrnd_node, n, s));
    RAPID_CHECK(upload(px->s_h1, vval_hash, n, s)); RAPID_CHECK(upload(px->s_len, vval_len, n, s));
    RAPID_CHECK(px->s_h2.reserve((size_t)n)); RAPID_CHECK(px->s_vr.reserve((size_t)n));
    if (vval_hash2) RAPID_CUDA(cudaMemcpyAsync(px->s_h2.p, vval_hash2, (size_t)n * 8, cudaMemcpyHostToDevice, s));
    else RAPID_CUDA(cudaMemsetAsync(px->s_h2.p, 0, (size_t)n * 8, s));
    k_px_pack<<<grid_for(n), TB, 0, s>>>(n, px->s_vrnd_round.p, px->s_vrnd_node.p, px->s_vr.p);
    RAPID_KERNEL_CHECK();
    RAPID_CHECK(px_rule_device(px, n, px->s_vr.p, px->s_h1.p, px->s_h2.p, px->s_len.p));
    RAPID_CUDA(cudaEventRecord(px->ev1, s));
    RAPID_CHECK(px_read_scal(px));
    cudaEventElapsedTime(&px->last_ms, px->ev0, px->ev1);
    if (px->h_sc.p->overflow) { set_error("internal: rule table overflow"); return RAPID_ECUDA; }
    *chosen_index = px->h_sc.p->chosen;
    return RAPID_OK;
}

int32_t rapid_px_phase1b(rapid_px* px, int64_t n, const int64_t* msg_cfg, const int32_t* rnd_round, const int32_t* rnd_node,
                         const int32_t* vrnd_round, const int32_t* vrnd_node, const uint64_t* vval_hash, const uint64_t* vval_hash2,
                         const int32_t* vval_len, int32_t* proposed, int64_t* trigger_index, uint64_t* cval_hash, uint64_t* cval_hash2,
                         int32_t* cval_len, int64_t* n_messages) {
    if (!px) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (n < 0 || n > 0x7ffffff0LL || (n && (!rnd_round || !rnd_node || !vrnd_round || !vrnd_node || !vval_hash || !vval_len))) { set_error("bad arguments"); return RAPID_EINVAL; }
    return px_timed(px, [&]() -> int32_t {
        WireMsgs m;
        RAPID_CHECK(px_stage(px, n, msg_cfg, rnd_round, rnd_node, vrnd_round, vrnd_node, nullptr, vval_hash, vval_hash2, vval_len, &m));
        return px_phase1b_msgs(px, m, proposed, trigger_index, cval_hash, cval_hash2, cval_len, n_messages);
    });
}

int32_t rapid_px_phase2b(rapid_px* px, int64_t n, const int64_t* msg_cfg, const int32_t* rnd_round, const int32_t* rnd_node,
                         const int32_t* sender, const uint64_t* hash, const uint64_t* hash2, const int32_t* len, int32_t* decided,
                         int64_t* decided_index, uint64_t* decided_hash, uint64_t* decided_hash2, int32_t* decided_len) {
    if (!px) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (n < 0 || n > 0x7ffffff0LL || (n && (!rnd_round || !rnd_node || !sender || !hash || !len))) { set_error("bad arguments"); return RAPID_EINVAL; }
    return px_timed(px, [&]() -> int32_t {
        WireMsgs m;
        RAPID_CHECK(px_stage(px, n, msg_cfg, rnd_round, rnd_node, nullptr, nullptr, sender, hash, hash2, len, &m));
        return px_phase2b_msgs(px, m, decided, decided_index, decided_hash, decided_hash2, decided_len);
    });
}

// the decoded messages of a wire handle (wire_internal.cuh): nothing uploaded
static int32_t px_wire_msgs(rapid_px* px, const rapid_wire* w, int32_t kind, WireMsgs* m) {
    if (!px) { set_error("NULL handle"); return RAPID_EINVAL; }
    RAPID_CHECK(wire_consensus_dev(w, kind, m));
    if (m->device != px->device) { set_error("px and wire live on different devices"); return RAPID_EINVAL; }
    return RAPID_OK;
}

int32_t rapid_px_phase1b_wire(rapid_px* px, const rapid_wire* w, int32_t* proposed, int64_t* trigger_index, uint64_t* cval_hash,
                              uint64_t* cval_hash2, int32_t* cval_len, int64_t* n_messages) {
    WireMsgs m;
    RAPID_CHECK(px_wire_msgs(px, w, RAPID_WIRE_PHASE1B, &m));
    return px_timed(px, [&]() -> int32_t {
        return px_phase1b_msgs(px, m, proposed, trigger_index, cval_hash, cval_hash2, cval_len, n_messages);
    });
}

int32_t rapid_px_phase2b_wire(rapid_px* px, const rapid_wire* w, int32_t* decided, int64_t* decided_index, uint64_t* decided_hash,
                              uint64_t* decided_hash2, int32_t* decided_len) {
    WireMsgs m;
    RAPID_CHECK(px_wire_msgs(px, w, RAPID_WIRE_PHASE2B, &m));
    return px_timed(px, [&]() -> int32_t {
        if (m.n > 0) {
            // a message of another configuration is dropped whatever its sender (:224); one of this configuration from an
            // endpoint outside the dictionary refuses the call before anything changes
            k_px2b_unknown_begin<<<1, 1, 0, px->stream>>>(px->sc.p);
            k_px2b_unknown<<<grid_for(m.n), TB, 0, px->stream>>>(m.n, m.cfg, px->cfg, m.sender, px->sc.p);
            RAPID_KERNEL_CHECK();
            RAPID_CHECK(px_read_scal(px));
            if (px->h_sc.p->unknown_sender != INT_MAX) {
                set_error("Phase2bMessage %d of the current configuration comes from an endpoint outside the dictionary", px->h_sc.p->unknown_sender);
                return RAPID_EINVAL;
            }
        }
        return px_phase2b_msgs(px, m, decided, decided_index, decided_hash, decided_hash2, decided_len);
    });
}

int32_t rapid_px_last_device_ms(const rapid_px* px, float* total_ms) {
    if (!px || !total_ms) return RAPID_EINVAL;
    *total_ms = px->last_ms;
    return RAPID_OK;
}

// ------------------------------------------------------------------ acceptors
int32_t rapid_pxa_create(rapid_pxa** out, int64_t cfg_id, int64_t n_acceptors, int64_t acceptor_begin, int32_t device) {
    if (!out || n_acceptors < 1 || n_acceptors > 0x7ffffff0LL || acceptor_begin < 0 || acceptor_begin + n_acceptors > 0x7ffffff0LL) { set_error("bad arguments"); return RAPID_EINVAL; }
    *out = nullptr;
    RAPID_CHECK(check_device(device));
    DeviceGuard g(device);
    rapid_pxa* a = new rapid_pxa();
    a->device = device; a->cfg = cfg_id; a->R = n_acceptors; a->begin = acceptor_begin;
    int32_t rc = RAPID_OK;
    do {
        if (cudaStreamCreateWithFlags(&a->stream, cudaStreamNonBlocking) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "stream", __FILE__, __LINE__); break; }
        const size_t R = (size_t)n_acceptors;
        if ((rc = a->rnd.reserve(R)) || (rc = a->vrnd.reserve(R)) || (rc = a->h1.reserve(R)) || (rc = a->h2.reserve(R)) || (rc = a->len.reserve(R))) break;
        if ((rc = a->reply.reserve(R)) || (rc = a->pos.reserve(R)) || (rc = a->o_sender.reserve(R)) || (rc = a->o_len.reserve(R)) ||
            (rc = a->o_vr.reserve(R)) || (rc = a->o_h1.reserve(R)) || (rc = a->o_h2.reserve(R))) break;
        if ((rc = a->total.reserve(1)) || (rc = a->h_total.reserve(1)) || (rc = a->bad.reserve(1))) break;
        k_pxa_init<<<grid_for(n_acceptors), TB, 0, a->stream>>>(n_acceptors, a->rnd.p, a->vrnd.p, a->h1.p, a->h2.p, a->len.p);
        cudaMemsetAsync(a->bad.p, 0, sizeof(int32_t), a->stream);
        if (cudaStreamSynchronize(a->stream) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "init", __FILE__, __LINE__); break; }
    } while (0);
    if (rc) { rapid_pxa_destroy(a); return rc; }
    *out = a;
    return RAPID_OK;
}

// every acceptor back to rnd = vrnd = (0, 0), vval = [] (Paxos ctor :82-85) for the next configuration
int32_t rapid_pxa_reset(rapid_pxa* a, int64_t cfg_id) {
    if (!a) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(a->device);
    a->cfg = cfg_id; a->last_kind = 0; a->n_out = 0;
    k_pxa_init<<<grid_for(a->R), TB, 0, a->stream>>>(a->R, a->rnd.p, a->vrnd.p, a->h1.p, a->h2.p, a->len.p);
    RAPID_KERNEL_CHECK();
    return RAPID_OK;
}

int32_t rapid_pxa_destroy(rapid_pxa* a) {
    if (!a) return RAPID_OK;
    DeviceGuard g(a->device);
    if (a->stream) { cudaStreamSynchronize(a->stream); cudaStreamDestroy(a->stream); }
    delete a;
    return RAPID_OK;
}

int32_t rapid_pxa_register_fast_round_votes(rapid_pxa* a, int64_t n, const int64_t* acceptor, const uint64_t* hash, const uint64_t* hash2,
                                            const int32_t* len) {
    if (!a) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (n < 0 || n > 0x7ffffff0LL || (n && (!acceptor || !hash || !len))) { set_error("bad arguments"); return RAPID_EINVAL; }
    if (n == 0) return RAPID_OK;
    DeviceGuard g(a->device);
    cudaStream_t s = a->stream;
    RAPID_CHECK(upload(a->s_acc, acceptor, n, s)); RAPID_CHECK(upload(a->s_h1, hash, n, s)); RAPID_CHECK(upload(a->s_len, len, n, s));
    if (hash2) RAPID_CHECK(upload(a->s_h2, hash2, n, s));
    RAPID_CHECK(a->win.reserve((size_t)a->R));
    RAPID_CUDA(cudaMemsetAsync(a->win.p, 0xff, (size_t)a->R * sizeof(int32_t), s));
    k_pxa_claim<<<grid_for(n), TB, 0, s>>>(n, a->s_acc.p, a->R, a->win.p, a->bad.p);
    k_pxa_register<<<grid_for(n), TB, 0, s>>>(n, a->s_acc.p, a->win.p, nullptr, a->s_h1.p, hash2 ? a->s_h2.p : nullptr, a->s_len.p,
                                              a->rnd.p, a->vrnd.p, a->h1.p, a->h2.p, a->len.p, a->bad.p);
    RAPID_KERNEL_CHECK();
    RAPID_CUDA(cudaMemcpyAsync(a->h_total.p, a->bad.p, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    if (*a->h_total.p) {
        cudaMemsetAsync(a->bad.p, 0, sizeof(int32_t), s);
        set_error("acceptor index out of range"); return RAPID_EINVAL;
    }
    return RAPID_OK;
}

int32_t rapid_pxa_register_fast_round_votes_cd(rapid_pxa* a, const rapid_cd* cd) {
    if (!a || !cd) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (a->device != cd->device) { set_error("acceptors and cd live on different devices"); return RAPID_EINVAL; }
    if (cd->raw) { set_error("RAW detectors do not announce proposals"); return RAPID_EINVAL; }
    if (cd->R != a->R) { set_error("detector has %lld receivers, handle has %lld acceptors", (long long)cd->R, (long long)a->R); return RAPID_EINVAL; }
    DeviceGuard g(a->device);
    RAPID_CUDA(cudaStreamSynchronize(cd->stream));            // the detector's outputs are produced on its own stream
    k_pxa_register<<<grid_for(a->R), TB, 0, a->stream>>>(a->R, nullptr, nullptr, cd->rflags.p, cd->out_h1.p, cd->out_h2.p, cd->out_len.p,
                                                         a->rnd.p, a->vrnd.p, a->h1.p, a->h2.p, a->len.p, a->bad.p);
    RAPID_KERNEL_CHECK();
    RAPID_CUDA(cudaStreamSynchronize(a->stream));
    return RAPID_OK;
}

static int32_t pxa_compact(rapid_pxa* a, bool with_values) {
    cudaStream_t s = a->stream;
    RAPID_CHECK(exclusive_scan_i32_to(a->reply.p, a->pos.p, a->R, a->scan_sums, s));
    k_pxa_gather1b<<<grid_for(a->R), TB, 0, s>>>(a->R, a->reply.p, a->pos.p, a->begin, a->vrnd.p, a->h1.p, a->h2.p, a->len.p, a->o_sender.p,
                                                 with_values ? a->o_vr.p : nullptr, a->o_h1.p, a->o_h2.p, a->o_len.p);
    k_pxa_total<<<1, 1, 0, s>>>(a->R, a->reply.p, a->pos.p, a->total.p);
    RAPID_KERNEL_CHECK();
    RAPID_CUDA(cudaMemcpyAsync(a->h_total.p, a->total.p, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    a->n_out = *a->h_total.p;
    return RAPID_OK;
}

int32_t rapid_pxa_phase1a(rapid_pxa* a, int64_t msg_cfg, int32_t round, int32_t node_index, int64_t* n_replies) {
    if (!a) { set_error("NULL handle"); return RAPID_EINVAL; }
    a->last_kind = 0; a->n_out = 0;
    if (n_replies) *n_replies = 0;
    if (msg_cfg != a->cfg) return RAPID_OK;                                          // :121-123
    DeviceGuard g(a->device);
    const int64_t rank = pack_rank(round, node_index);
    // answers carry the vrnd / vval each acceptor held when it answered, so they are gathered in the same pass
    k_pxa_phase1a<<<grid_for(a->R), TB, 0, a->stream>>>(a->R, rank, a->has_silent ? a->silent.p : nullptr, a->rnd.p, a->reply.p);
    RAPID_KERNEL_CHECK();
    RAPID_CHECK(pxa_compact(a, true));
    a->last_kind = 1; a->last_rank = rank;
    if (n_replies) *n_replies = a->n_out;
    return RAPID_OK;
}

int32_t rapid_pxa_phase2a(rapid_pxa* a, int64_t msg_cfg, int32_t round, int32_t node_index, uint64_t hash, uint64_t hash2, int32_t len,
                          int64_t* n_accepted) {
    if (!a) { set_error("NULL handle"); return RAPID_EINVAL; }
    a->last_kind = 0; a->n_out = 0;
    if (n_accepted) *n_accepted = 0;
    if (msg_cfg != a->cfg) return RAPID_OK;                                          // :199-201
    DeviceGuard g(a->device);
    const int64_t rank = pack_rank(round, node_index);
    k_pxa_phase2a<<<grid_for(a->R), TB, 0, a->stream>>>(a->R, rank, hash, hash2, len, a->has_silent ? a->silent.p : nullptr, a->rnd.p, a->vrnd.p, a->h1.p, a->h2.p, a->len.p, a->reply.p);
    RAPID_KERNEL_CHECK();
    RAPID_CHECK(pxa_compact(a, false));
    a->last_kind = 2; a->last_rank = rank; a->last_h1 = hash; a->last_h2 = hash2; a->last_len = len;
    if (n_accepted) *n_accepted = a->n_out;
    return RAPID_OK;
}

int32_t rapid_px_phase1b_from_acceptor_shards(rapid_px* px, const rapid_pxa* const* shards, int32_t n_shards, rapid_comm* comm,
                                              uint64_t perm_seed, int32_t* proposed, int64_t* trigger_index, uint64_t* cval_hash,
                                              uint64_t* cval_hash2, int32_t* cval_len, int64_t* n_messages) {
    if (!px) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (comm && comm->device != px->device) { set_error("comm and px live on different devices"); return RAPID_EINVAL; }
    return px_timed(px, [&]() -> int32_t {
        PxaAnswers a;
        RAPID_CHECK(px_gather_shards(px, shards, n_shards, comm, 1, &a));
        const int32_t* order = nullptr;
        RAPID_CHECK(px_arrival_order(px, a.sender, a.n, perm_seed, &order));
        if (order) {
            cudaStream_t s = px->stream;
            const int64_t n = a.n;
            RAPID_CHECK(px->g_vr.reserve((size_t)n)); RAPID_CHECK(px->g_h1.reserve((size_t)n));
            RAPID_CHECK(px->g_h2.reserve((size_t)n)); RAPID_CHECK(px->g_len.reserve((size_t)n));
            k_px_gather<int64_t><<<grid_for(n), TB, 0, s>>>(n, order, a.vrnd, px->g_vr.p);
            k_px_gather<uint64_t><<<grid_for(n), TB, 0, s>>>(n, order, a.h1, px->g_h1.p);
            k_px_gather<uint64_t><<<grid_for(n), TB, 0, s>>>(n, order, a.h2, px->g_h2.p);
            k_px_gather<int32_t><<<grid_for(n), TB, 0, s>>>(n, order, a.len, px->g_len.p);
            RAPID_KERNEL_CHECK();
            a.vrnd = px->g_vr.p; a.h1 = px->g_h1.p; a.h2 = px->g_h2.p; a.len = px->g_len.p;
        }
        return px_phase1b_device(px, a.n, nullptr, nullptr, a.rank, a.vrnd, a.h1, a.h2, a.len, proposed, trigger_index, cval_hash,
                                 cval_hash2, cval_len, n_messages);
    });
}

int32_t rapid_px_phase2b_from_acceptor_shards(rapid_px* px, const rapid_pxa* const* shards, int32_t n_shards, rapid_comm* comm,
                                              uint64_t perm_seed, int32_t* decided, int64_t* decided_index, uint64_t* decided_hash,
                                              uint64_t* decided_hash2, int32_t* decided_len) {
    if (!px) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (comm && comm->device != px->device) { set_error("comm and px live on different devices"); return RAPID_EINVAL; }
    return px_timed(px, [&]() -> int32_t {
        PxaAnswers a;
        RAPID_CHECK(px_gather_shards(px, shards, n_shards, comm, 2, &a));
        const int32_t* order = nullptr;
        RAPID_CHECK(px_arrival_order(px, a.sender, a.n, perm_seed, &order));
        return px_phase2b_device(px, a.n, nullptr, nullptr, a.rank, order ? px->g_sender.p : a.sender, nullptr, nullptr, nullptr, a.v_h1,
                                 a.v_h2, a.v_len, decided, decided_index, decided_hash, decided_hash2, decided_len);
    });
}

int32_t rapid_pxa_set_silent(rapid_pxa* a, const uint8_t* silent) {
    if (!a) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(a->device);
    if (!silent) { a->has_silent = false; return RAPID_OK; }
    RAPID_CHECK(upload(a->silent, silent, a->R, a->stream));
    RAPID_CUDA(cudaStreamSynchronize(a->stream));                                    // the host array may go away after the call
    a->has_silent = true;
    return RAPID_OK;
}

int32_t rapid_pxa_find_value(const rapid_pxa* a, uint64_t hash, uint64_t hash2, int32_t len, int64_t* acceptor) {
    if (!a || !acceptor) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(a->device);
    rapid_pxa* m = const_cast<rapid_pxa*>(a);                                        // scratch only; no acceptor state changes
    cudaStream_t s = m->stream;
    RAPID_CHECK(m->found.reserve(1)); RAPID_CHECK(m->h_found.reserve(1));
    const unsigned long long none = (unsigned long long)a->R;
    RAPID_CUDA(cudaMemcpyAsync(m->found.p, &none, sizeof(none), cudaMemcpyHostToDevice, s));
    k_pxa_find<<<grid_for(a->R), TB, 0, s>>>(a->R, hash, hash2, len, a->h1.p, a->h2.p, a->len.p, m->found.p);
    RAPID_KERNEL_CHECK();
    RAPID_CUDA(cudaMemcpyAsync(m->h_found.p, m->found.p, sizeof(none), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    *acceptor = *m->h_found.p < none ? (int64_t)*m->h_found.p : -1;
    return RAPID_OK;
}

int32_t rapid_pxa_read(const rapid_pxa* a, int64_t acceptor, int32_t* ranks, uint64_t* hash, uint64_t* hash2, int32_t* len) {
    if (!a || acceptor < 0 || acceptor >= a->R) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(a->device);
    int64_t r[2]; uint64_t h[2]; int32_t l;
    RAPID_CUDA(cudaStreamSynchronize(a->stream));
    RAPID_CUDA(cudaMemcpy(&r[0], a->rnd.p + acceptor, 8, cudaMemcpyDeviceToHost));
    RAPID_CUDA(cudaMemcpy(&r[1], a->vrnd.p + acceptor, 8, cudaMemcpyDeviceToHost));
    RAPID_CUDA(cudaMemcpy(&h[0], a->h1.p + acceptor, 8, cudaMemcpyDeviceToHost));
    RAPID_CUDA(cudaMemcpy(&h[1], a->h2.p + acceptor, 8, cudaMemcpyDeviceToHost));
    RAPID_CUDA(cudaMemcpy(&l, a->len.p + acceptor, 4, cudaMemcpyDeviceToHost));
    if (ranks) { ranks[0] = rank_round(r[0]); ranks[1] = rank_node(r[0]); ranks[2] = rank_round(r[1]); ranks[3] = rank_node(r[1]); }
    if (hash) *hash = h[0];
    if (hash2) *hash2 = h[1];
    if (len) *len = l;
    return RAPID_OK;
}

}  // extern "C"
