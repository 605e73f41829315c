// FastPaxos fast-round vote tally (rapid/src/main/java/com/vrg/rapid/FastPaxos.java:125-156) on the device,
// plus the sharded (multi-GPU) variant: per-rank proposal-hash histograms combined with one NCCL all-reduce.
//
// The Java keeps HashMap<List<Endpoint>, AtomicInteger> and hashes the whole endpoint list for every vote
// (O(#cut) per vote).  Here a proposal is its 128-bit order-independent fingerprint + length (computed once
// per proposer by the cut-detection kernels).  One cooperative kernel tallies the votes of a call, whether they
// come from host arrays or straight from a detector's outputs: votes are de-duplicated per sender with an
// atomicMin "first index" table, counted in an open-addressing table with warp-aggregated atomics, and the
// exact decision point (the vote at which a count reaches N - floor((N-1)/4)) is recovered with per-block
// counts and in-block scans so that votesReceived / count at the moment of decision match the sequential
// reference.
#include <cooperative_groups.h>
#include <dlfcn.h>

#include <algorithm>
#include <climits>
#include <cstdlib>

#include "cd_internal.cuh"
#include "nccl_api.cuh"
#include "wire_internal.cuh"

namespace cg = cooperative_groups;

namespace rapid {

struct FPState {
    int32_t decided;
    int32_t decided_entry;
    int32_t votes_received;
    int32_t n_cand;
    int32_t cand[8];
    int32_t i_star;
    int32_t bad_sender;     // largest index of a vote whose sender is outside [0, sender_cap) (-1: none)
    int32_t n_entries;      // table entries created since the last reset (listed in FP::entries)
    int32_t n_call;         // entries that received votes in the call in flight (listed in FP::call_list)
    int32_t ticket;         // "last block done" counter of k_fp_tally
    int32_t calls;          // rapid_fp_tally_cd[_async] calls since the last reset
    int32_t decided_call;   // index of the call that decided (-1: undecided)
};

struct FPResult {
    int32_t decided, len, count, received;   // decided = -1: refused, more than 8 proposals reached the quorum
    uint64_t h1, h2;
    int32_t decided_call, bad_sender;         // bad_sender >= 0: refused, FPState::bad_sender
};
struct FP {
    int device = 0;
    bool decided_host = false;            // host mirror of FPState::decided
    DevBuf<unsigned char> d_res_raw;      // FPResult on the device
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    int64_t cfg = 0, N = 0, Q = 0, sender_cap = 0;
    uint32_t T = 0;                       // table capacity (power of two)
    DevBuf<int32_t> seen;                 // [sender_cap] INT_MAX = not voted, -1 = voted, else first index in the call
    DevBuf<int32_t> t_state, t_len, t_count, t_call;
    DevBuf<uint64_t> t_h1, t_h2;
    DevBuf<int32_t> ent;                  // per-vote scratch
    DevBuf<int32_t> entries, call_list;   // [T] created entries / entries voted for in the call in flight
    DevBuf<int32_t> blk_cnt;              // [8][grid] per-block vote counts of the quorum candidates (k_fp_tally)
    int tally_grid = 0;                   // co-resident blocks of the cooperative tally kernel
    rapid_comm* pending_comm = nullptr;   // what the last enqueued rapid_fp_tally_cd[_async] was called with
    const rapid_cd* pending_cd = nullptr;
    DevBuf<FPState> st;
    PinnedBuf<FPState> h_st;
    // staging for host-array votes
    DevBuf<int32_t> v_sender, v_len;
    DevBuf<int64_t> v_cfg;
    DevBuf<uint64_t> v_h1, v_h2;
    // sharded tally
    DevBuf<int32_t> hist;                 // [65536] (refinement path)
    DevBuf<unsigned long long> sumbuf;    // [(4096 + 1) * 8] the single all-reduce buffer
    DevBuf<unsigned long long> mm;        // [8] max / ~min verification words
    PinnedBuf<unsigned long long> h_mm;
    PinnedBuf<unsigned char> h_res_raw;
    float last_ms = 0.f;
    int32_t last_launches = 0;
};

// ------------------------------------------------------------------ NCCL through dlopen (nccl_api.cuh)
NcclApi g_nccl;

int32_t load_nccl() {
    if (g_nccl.lib) return RAPID_OK;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    void* h = nullptr;
    for (const char* n : names) { h = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (h) break; }
    if (!h) { set_error("cannot dlopen libnccl.so.2: %s", dlerror()); return RAPID_ENCCL; }
    NcclApi a;
    a.lib = h;
    a.GetUniqueId = (int (*)(nccl_uid*))dlsym(h, "ncclGetUniqueId");
    a.CommInitRank = (int (*)(nccl_comm*, int, nccl_uid, int))dlsym(h, "ncclCommInitRank");
    a.CommDestroy = (int (*)(nccl_comm))dlsym(h, "ncclCommDestroy");
    a.AllReduce = (int (*)(const void*, void*, size_t, int, int, nccl_comm, cudaStream_t))dlsym(h, "ncclAllReduce");
    a.AllGather = (int (*)(const void*, void*, size_t, int, nccl_comm, cudaStream_t))dlsym(h, "ncclAllGather");
    a.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
    if (!a.GetUniqueId || !a.CommInitRank || !a.CommDestroy || !a.AllReduce) { set_error("libnccl lacks required symbols"); return RAPID_ENCCL; }
    g_nccl = a;
    return RAPID_OK;
}

// ------------------------------------------------------------------ kernels
// a new FastPaxos instance on the same buffers, one launch
__global__ void k_fp_reset(int64_t sender_cap, int32_t* __restrict__ seen, uint32_t T, int32_t* __restrict__ t_state,
                           int32_t* __restrict__ t_count, int32_t* __restrict__ t_call, FPState* __restrict__ st);

__global__ void k_fp_fill(int32_t* p, int64_t n, int32_t v) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

__global__ void k_fp_reset(int64_t sender_cap, int32_t* __restrict__ seen, uint32_t T, int32_t* __restrict__ t_state,
                           int32_t* __restrict__ t_count, int32_t* __restrict__ t_call, FPState* __restrict__ st) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < sender_cap) seen[i] = INT_MAX;
    if (i < (int64_t)T) { t_state[i] = 0; t_count[i] = 0; t_call[i] = 0; }
    if (i == 0) {
        st->decided = 0; st->decided_entry = 0; st->votes_received = 0; st->n_cand = 0; st->i_star = INT_MAX; st->bad_sender = -1;
        st->n_entries = 0; st->n_call = 0; st->ticket = 0; st->calls = 0; st->decided_call = -1;
    }
}

__device__ __forceinline__ uint32_t fp_slot_hash(uint64_t h1, uint64_t h2, int32_t len) {
    return (uint32_t)(splitmix64(h1 ^ rotl64(h2, 21) ^ (uint64_t)(uint32_t)len) >> 32);
}

// ---- sharded tally: radix histogram over the proposal fingerprints, restricted to a prefix -----------------------
// level l looks at 16-bit digit l of the 128-bit string (h1 high..low, then h2 high..low); entries must match the
// `prefix` digits chosen so far.
__device__ __forceinline__ uint32_t fp_digit(uint64_t h1, uint64_t h2, int level) {
    const uint64_t w = level < 4 ? h1 : h2;
    return (uint32_t)(w >> (48 - 16 * (level & 3))) & 0xffffu;
}
struct Prefix { uint32_t d[8]; int n; };

__global__ void k_fp_hist(uint32_t T, const int32_t* __restrict__ t_state, const uint64_t* __restrict__ t_h1,
                          const uint64_t* __restrict__ t_h2, const int32_t* __restrict__ t_count, Prefix pf,
                          int32_t* __restrict__ hist) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= T || t_state[e] != 2) return;
    const int32_t c = t_count[e];
    if (c == 0) return;
    const uint64_t h1 = t_h1[e], h2 = t_h2[e];
    for (int l = 0; l < pf.n; ++l) if (fp_digit(h1, h2, l) != pf.d[l]) return;
    atomicAdd(&hist[fp_digit(h1, h2, pf.n)], c);
}

__global__ void k_fp_hist_cand(const int32_t* __restrict__ hist, int32_t Q, FPState* __restrict__ st) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= 65536) return;
    if (hist[b] >= Q) {
        const int32_t at = atomicAdd(&st->n_cand, 1);
        if (at < 8) st->cand[at] = (int32_t)b;
    }
}

// max / ~min of (h1, h2, len) over the local entries matching the prefix (identity 0 for ranks without one)
__global__ void k_fp_minmax(uint32_t T, const int32_t* __restrict__ t_state, const uint64_t* __restrict__ t_h1,
                            const uint64_t* __restrict__ t_h2, const int32_t* __restrict__ t_len,
                            const int32_t* __restrict__ t_count, Prefix pf, unsigned long long* __restrict__ mm) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= T || t_state[e] != 2 || t_count[e] == 0) return;
    const uint64_t h1 = t_h1[e], h2 = t_h2[e];
    for (int l = 0; l < pf.n; ++l) if (fp_digit(h1, h2, l) != pf.d[l]) return;
    const unsigned long long len = (unsigned long long)(uint32_t)t_len[e];
    atomicMax(&mm[0], (unsigned long long)h1); atomicMax(&mm[1], ~(unsigned long long)h1);
    atomicMax(&mm[2], (unsigned long long)h2); atomicMax(&mm[3], ~(unsigned long long)h2);
    atomicMax(&mm[4], len);                    atomicMax(&mm[5], ~len);
}

__global__ void k_fp_begin(FPState* st) {
    st->n_cand = 0; st->i_star = INT_MAX; st->bad_sender = -1;
}

// ---- sharded tally, the single all-reduce: per 12-bit bucket of the fingerprint, SUMS of (count, h1 hi/lo, h2 hi/lo, len,
// check hi/lo) weighted by the vote counts.  After ncclAllReduce(sum) a bucket that reached the quorum and holds ONE
// proposal gives it back by exact division, and the independent check word proves there was only one (two different
// proposals averaging to integers would have to collide on a 64-bit mix as well).
constexpr int SUM_BUCKETS = 4096, SUM_WORDS = 8;

__device__ __forceinline__ uint64_t fp_check_word(uint64_t h1, uint64_t h2, uint64_t len) {
    return splitmix64(h1 ^ rotl64(h2, 17) ^ (len * 0x9E3779B97F4A7C15ULL));
}

struct FPSumResult {
    FPResult r;
    int32_t ambiguous;       // a bucket reached the quorum but holds more than one proposal
    int32_t pad;
};

// one block: initialise the result, then look for the bucket that reached the quorum
__global__ void __launch_bounds__(1024) k_fp_decide_sum(const unsigned long long* __restrict__ buf, unsigned long long Q,
                                                        FPSumResult* __restrict__ out, FPState* __restrict__ st) {
    __shared__ int32_t s_call;
    if (threadIdx.x == 0) {
        out->r.decided = 0; out->r.len = 0; out->r.count = 0; out->r.h1 = 0; out->r.h2 = 0;
        out->r.received = (int32_t)buf[(size_t)SUM_BUCKETS * SUM_WORDS];
        out->r.decided_call = st->decided_call; out->r.bad_sender = -1;
        out->ambiguous = 0; out->pad = 0;
        s_call = st->calls;
        st->calls = s_call + 1;
    }
    __syncthreads();
    for (int b = threadIdx.x; b < SUM_BUCKETS; b += blockDim.x) {
        const unsigned long long* w = buf + (size_t)b * SUM_WORDS;
        const unsigned long long c = w[0];
        if (c < Q || c == 0) continue;
        bool ok = true;
        for (int q = 1; q < SUM_WORDS; ++q) ok = ok && (w[q] % c == 0);
        uint64_t h1 = 0, h2 = 0, len = 0;
        if (ok) {
            const uint64_t a1 = w[1] / c, a2 = w[2] / c, b1 = w[3] / c, b2 = w[4] / c;
            len = w[5] / c;
            ok = a1 <= 0xFFFFFFFFull && a2 <= 0xFFFFFFFFull && b1 <= 0xFFFFFFFFull && b2 <= 0xFFFFFFFFull && len <= 0x7FFFFFFFull;
            h1 = (a1 << 32) | a2; h2 = (b1 << 32) | b2;
            if (ok) {
                const uint64_t m = fp_check_word(h1, h2, len);
                ok = (w[6] / c == (m >> 32)) && (w[7] / c == (m & 0xFFFFFFFFull)) && ((h1 >> 52) == (uint64_t)b);
            }
        }
        if (ok) {
            out->r.decided = 1; out->r.h1 = h1; out->r.h2 = h2; out->r.len = (int32_t)len; out->r.count = (int32_t)c;
            // remember the decision locally so that later votes are ignored (:138)
            if (!st->decided) { st->decided_call = s_call; out->r.decided_call = s_call; }
            st->decided = 1; st->decided_entry = -1;
        } else {
            out->ambiguous = 1;
        }
    }
}

// ==================================================================================================================
// k_fp_tally<ARRAY>: the fast-round tally of one call in ONE cooperative launch, for votes from either source.
//
// ARRAY = false: every receiver that announced in the last batch votes for its proposal (FastPaxos.propose :94-108), in
//   receiver order (= arrival order on one GPU).  Senders are unique by construction, so "first vote of a sender" is just
//   "has not voted in an earlier call".
// ARRAY = true: vote i is (sender[i], vcfg[i], h1v[i], h2v[i], lenv[i]) in arrival order, as the host handed them over.  A
//   sender may vote several times; only its first vote of this configuration counts (:126, :134).
// WIRE = true (with ARRAY): the votes are decoded messages (rapid_fp_tally_wire), whose sender is -1 when the dictionary does
//   not hold it.  A vote of another configuration is dropped first (:126), so only a vote of THIS configuration from a sender
//   outside [0, sender_cap) refuses the call.
// Phases (grid barriers in between, every block owns a CONTIGUOUS range of votes so that arrival order is block order):
//   V  (ARRAY) a sender outside [0, sender_cap) refuses the whole call before anything is marked (WIRE: of this configuration)
//   F  (ARRAY) the first vote of every sender in this call: atomicMin of its index into seen[] (-1, voted earlier, stays)
//   A  find-or-insert the proposal of every first vote (warp- and block-aggregated counts -> t_call); the add that takes a
//      proposal over the quorum nominates it as a candidate
//   C  only if there is a candidate: the exact vote i* at which its running count reaches the quorum (per-block counts,
//      prefix over blocks, in-block scan) — votes after i* are ignored, as the sequential reference would (:138)
//   D  apply: votesReceived, counts, seen marks for the votes with index <= i*; the first votes after i* are unmarked
//   tail (last block): decision + result record, per-call scratch re-armed
// More than 8 proposals crossing the quorum in one call refuses it: C is skipped and D counts nothing, so the refused call
// leaves no trace and does not decide.  Once decided, a call changes nothing and reports the stored result.
// direct != 0 (sharded tally, detector votes only): no arrival order across ranks — counts go straight to t_count and
// phase S adds this rank's table to the all-reduce buffer.
// ==================================================================================================================
constexpr int TALLY_THREADS = 256;

struct TallyArgs {
    int64_t R;                  // votes
    int64_t rbegin;             // detector votes: receiver i votes iff rflags[i] & RF_ANN_NOW, as sender ring0[rbegin + i]
    const uint32_t* rflags;
    const int32_t* ring0;
    const int32_t* sender;      // array votes: vote i comes from sender[i] for configuration vcfg[i] (vcfg NULL: cfg)
    const int64_t* vcfg;
    int64_t cfg;
    const uint64_t* h1v;
    const uint64_t* h2v;        // array votes: NULL means 0
    const int32_t* lenv;        // array votes: NULL means 0
    int64_t sender_cap;
    int32_t* seen;
    uint32_t T;
    int32_t* t_state;
    uint64_t* t_h1;
    uint64_t* t_h2;
    int32_t* t_len;
    int32_t* t_count;
    int32_t* t_call;
    int32_t* ent;
    int32_t* entries;
    int32_t* call_list;
    int32_t* blk_cnt;
    FPState* st;
    int32_t Q;
    int direct;
    unsigned long long* sumbuf;
    FPResult* out;
};

__device__ __forceinline__ int32_t fp_find_or_insert(const TallyArgs& a, uint64_t h1, uint64_t h2, int32_t len) {
    uint32_t pos = fp_slot_hash(h1, h2, len) & (a.T - 1);
    for (;;) {
        int32_t state = *(volatile int32_t*)&a.t_state[pos];              // published entries need no atomic
        if (state == 0) state = atomicCAS(&a.t_state[pos], 0, 1);
        if (state == 0) {                                                 // claimed an empty entry: publish the key
            a.t_h1[pos] = h1; a.t_h2[pos] = h2; a.t_len[pos] = len;
            __threadfence();
            atomicExch(&a.t_state[pos], 2);
            a.entries[atomicAdd(&a.st->n_entries, 1)] = (int32_t)pos;
            return (int32_t)pos;
        }
        while (state == 1) state = atomicAdd(&a.t_state[pos], 0);          // another warp is publishing
        __threadfence();
        if (a.t_h1[pos] == h1 && a.t_h2[pos] == h2 && a.t_len[pos] == len) return (int32_t)pos;
        pos = (pos + 1) & (a.T - 1);
    }
}

// add c votes of this call to entry e; nominate it if THIS add takes it over the quorum
__device__ __forceinline__ void fp_add_call(const TallyArgs& a, int32_t e, int32_t c) {
    if (a.direct) { atomicAdd(&a.t_count[e], c); return; }
    const int32_t old = atomicAdd(&a.t_call[e], c);
    if (old == 0) a.call_list[atomicAdd(&a.st->n_call, 1)] = e;
    const int32_t before = a.t_count[e] + old;
    if (before < a.Q && before + c >= a.Q) {
        const int32_t at = atomicAdd(&a.st->n_cand, 1);
        if (at < 8) a.st->cand[at] = e;                  // more than 8 refuse the call
    }
}

__device__ __forceinline__ int32_t tally_block_scan(int32_t v, int32_t* warp_sums, int32_t* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int32_t x = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += x;
    }
    __syncthreads();
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        int32_t s = lane < (TALLY_THREADS >> 5) ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int32_t x = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += x;
        }
        if (lane < (TALLY_THREADS >> 5)) warp_sums[lane] = s;
    }
    __syncthreads();
    *total = warp_sums[(TALLY_THREADS >> 5) - 1];
    return (wid ? warp_sums[wid - 1] : 0) + inc - v;
}

template <bool ARRAY, bool WIRE = false>
__global__ void __launch_bounds__(TALLY_THREADS) k_fp_tally(const TallyArgs a) {
    cg::grid_group grid = cg::this_grid();
    __shared__ int32_t s_key[16], s_val[16], s_recv, s_last;
    __shared__ int32_t warp_sums[TALLY_THREADS / 32];
    const int t = threadIdx.x, G = gridDim.x, bid = blockIdx.x;
    const int64_t per = ((a.R + G - 1) / G + TALLY_THREADS - 1) / TALLY_THREADS * TALLY_THREADS;
    const int64_t c0 = min(a.R, (int64_t)bid * per), c1 = min(a.R, c0 + per);
    const bool direct = !ARRAY && a.direct;
    bool skip = a.st->decided != 0;                       // :138 — everything after the decision is ignored

    auto block_flush = [&](bool to_count) {               // block-level partial counts -> global
        __syncthreads();
        if (t < 16 && s_key[t] >= 0) {
            if (to_count) atomicAdd(&a.t_count[s_key[t]], s_val[t]);
            else fp_add_call(a, s_key[t], s_val[t]);
        }
        __syncthreads();
        if (t < 16) { s_key[t] = -1; s_val[t] = 0; }
        __syncthreads();
    };
    auto block_add = [&](int32_t e, int32_t c, bool to_count) {   // called by one lane per (warp, entry)
        int slot = -1;
        for (int q = 0; q < 16; ++q) {
            const int32_t k = atomicCAS(&s_key[q], -1, e);
            if (k == -1 || k == e) { slot = q; break; }
        }
        if (slot >= 0) atomicAdd(&s_val[slot], c);
        else if (to_count) atomicAdd(&a.t_count[e], c);           // more than 16 distinct proposals in one block
        else fp_add_call(a, e, c);
    };

    if (ARRAY && !skip) {
        // ---- V: a sender outside the table refuses the call; nothing is marked yet, so nothing has to be undone ---------------
        for (int64_t i = c0 + t; i < c1; i += TALLY_THREADS) {
            const int32_t s = a.sender[i];
            if ((s < 0 || s >= a.sender_cap) && (!WIRE || a.vcfg[i] == a.cfg)) atomicMax(&a.st->bad_sender, (int32_t)i);
        }
        grid.sync();
        skip = *(volatile int32_t*)&a.st->bad_sender >= 0;
        if (!skip) {
            // ---- F: the first vote of every sender in this call (votesReceived.contains(sender), :134) ----------------------------
            for (int64_t i = c0 + t; i < c1; i += TALLY_THREADS)
                if (!a.vcfg || a.vcfg[i] == a.cfg) atomicMin(&a.seen[a.sender[i]], (int32_t)i);   // :126; -1 (voted earlier) stays
            grid.sync();
        }
    }
    if (t < 16) { s_key[t] = -1; s_val[t] = 0; }
    if (t == 0) s_recv = 0;
    __syncthreads();
    if (!skip) {
        // ---- A: one table probe per distinct fingerprint per warp ------------------------------------------------------------
        for (int64_t base = c0; base < c1; base += TALLY_THREADS) {
            const int64_t i = base + t;
            bool valid = false;
            uint64_t h1 = 0, h2 = 0;
            int32_t len = 0, sender = -1;
            if (ARRAY) {
                valid = i < c1 && (!a.vcfg || a.vcfg[i] == a.cfg) && a.seen[a.sender[i]] == (int32_t)i;
                if (valid) { h1 = a.h1v[i]; h2 = a.h2v ? a.h2v[i] : 0; len = a.lenv ? a.lenv[i] : 0; }
            } else if (i < c1 && (a.rflags[i] & RF_ANN_NOW)) {
                sender = a.ring0[a.rbegin + i];
                if (sender >= 0 && sender < a.sender_cap && a.seen[sender] != -1) {
                    valid = true;
                    h1 = a.h1v[i]; h2 = a.h2v[i]; len = a.lenv[i];
                }
            }
            int32_t e = -1;
            const unsigned active = __ballot_sync(0xffffffffu, valid);
            if (valid) {
                const unsigned same = __match_any_sync(active, h1 ^ rotl64(h2, 21) ^ ((uint64_t)(uint32_t)len << 1));
                const int leader = __ffs(same) - 1;
                if ((t & 31) == leader) e = fp_find_or_insert(a, h1, h2, len);
                e = __shfl_sync(same, e, leader);
                const uint64_t lh1 = __shfl_sync(same, h1, leader), lh2 = __shfl_sync(same, h2, leader);
                const int32_t llen = __shfl_sync(same, len, leader);
                const bool mine = lh1 == h1 && lh2 == h2 && llen == len;
                if (!mine) e = fp_find_or_insert(a, h1, h2, len);           // folded-key collision inside the warp (astronomically rare)
                const unsigned grp = __match_any_sync(same, e);             // the leader's group minus the collided lanes, per entry
                if ((t & 31) == __ffs(grp) - 1) block_add(e, __popc(grp), direct);
                if (direct) a.seen[sender] = -1;
            }
            if (i < c1) a.ent[i] = e;
            if (direct && (t & 31) == 0 && active) atomicAdd(&s_recv, __popc(active));
        }
        block_flush(direct);
        if (direct && t == 0 && s_recv) atomicAdd(&a.st->votes_received, s_recv);
    }
    if (direct) {
        // ---- S: this rank's table -> the all-reduce buffer (count-weighted sums per 12-bit bucket of the fingerprint) ------
        grid.sync();
        const int32_t ne = *(volatile int32_t*)&a.st->n_entries;
        if (bid == 0 && t == 0) a.sumbuf[(size_t)SUM_BUCKETS * SUM_WORDS] = (unsigned long long)*(volatile int32_t*)&a.st->votes_received;
        for (int32_t q = bid * TALLY_THREADS + t; q < ne; q += G * TALLY_THREADS) {
            const int32_t e = a.entries[q];
            const unsigned long long c = (unsigned long long)a.t_count[e];
            if (c == 0) continue;
            const uint64_t h1 = a.t_h1[e], h2 = a.t_h2[e], len = (uint64_t)(uint32_t)a.t_len[e], m = fp_check_word(h1, h2, len);
            unsigned long long* b = a.sumbuf + (size_t)(h1 >> 52) * SUM_WORDS;
            atomicAdd(b + 0, c);
            atomicAdd(b + 1, c * (h1 >> 32)); atomicAdd(b + 2, c * (h1 & 0xFFFFFFFFull));
            atomicAdd(b + 3, c * (h2 >> 32)); atomicAdd(b + 4, c * (h2 & 0xFFFFFFFFull));
            atomicAdd(b + 5, c * len);
            atomicAdd(b + 6, c * (m >> 32)); atomicAdd(b + 7, c * (m & 0xFFFFFFFFull));
        }
        return;
    }
    grid.sync();
    const int32_t nominated = skip ? 0 : *(volatile int32_t*)&a.st->n_cand;
    const bool too_many = nominated > 8;
    const int32_t n_cand = too_many ? 0 : nominated;
    int64_t limit = too_many ? -1 : INT64_MAX;
    if (n_cand > 0) {
        // ---- C: the vote at which a candidate's running count reaches the quorum ------------------------------------------------
        for (int c = 0; c < n_cand; ++c) {
            const int32_t e = ((volatile FPState*)a.st)->cand[c];
            int32_t mine = 0;
            for (int64_t i = c0 + t; i < c1; i += TALLY_THREADS) mine += a.ent[i] == e ? 1 : 0;
            int32_t total;
            tally_block_scan(mine, warp_sums, &total);
            if (t == 0) a.blk_cnt[(size_t)c * G + bid] = total;
        }
        grid.sync();
        for (int c = 0; c < n_cand; ++c) {
            const int32_t e = ((volatile FPState*)a.st)->cand[c];
            const int32_t need = a.Q - a.t_count[e];                       // >= 1: it was below the quorum before this call
            int32_t before = 0;
            for (int q = t; q < bid; q += TALLY_THREADS) before += *(volatile int32_t*)&a.blk_cnt[(size_t)c * G + q];
            int32_t prefix;
            tally_block_scan(before, warp_sums, &prefix);
            const int32_t own = *(volatile int32_t*)&a.blk_cnt[(size_t)c * G + bid];
            if (!(prefix < need && need <= prefix + own)) continue;       // uniform across the block
            for (int64_t base = c0; base < c1; base += TALLY_THREADS) {
                const int64_t i = base + t;
                const int32_t f = (i < c1 && a.ent[i] == e) ? 1 : 0;
                int32_t total;
                const int32_t off = tally_block_scan(f, warp_sums, &total);
                if (f && prefix + off + 1 == need) atomicMin(&a.st->i_star, (int32_t)i);
                prefix += total;
            }
        }
        grid.sync();
        limit = (int64_t)*(volatile int32_t*)&a.st->i_star;
    }
    if (!skip) {
        // ---- D: votesReceived.add(sender) :141, count :142-144 for the votes up to the decision ------------------------------
        if (t == 0) s_recv = 0;
        __syncthreads();
        for (int64_t base = c0; base < c1; base += TALLY_THREADS) {
            const int64_t i = base + t;
            const int32_t e = i < c1 ? a.ent[i] : -1;
            const bool counted = e >= 0 && i <= limit;
            if (counted) a.seen[ARRAY ? a.sender[i] : a.ring0[a.rbegin + i]] = -1;
            else if (ARRAY && e >= 0) a.seen[a.sender[i]] = INT_MAX;          // a first vote after the decision: ignored (:138)
            const unsigned m = __ballot_sync(0xffffffffu, counted);
            if (counted) {
                const unsigned same = __match_any_sync(m, e);
                if ((t & 31) == __ffs(same) - 1) block_add(e, __popc(same), true);
            }
            if ((t & 31) == 0 && m) atomicAdd(&s_recv, __popc(m));
        }
        block_flush(true);
        if (t == 0 && s_recv) atomicAdd(&a.st->votes_received, s_recv);
    }
    // ---- tail: the last block publishes the outcome and re-arms the per-call scratch ---------------------------------------------
    __syncthreads();
    if (t == 0) { __threadfence(); s_last = atomicAdd(&a.st->ticket, 1) == G - 1; }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    volatile FPState* st = a.st;
    const int32_t nc = st->n_call;
    for (int32_t q = t; q < nc; q += TALLY_THREADS) a.t_call[a.call_list[q]] = 0;
    if (t == 0) {
        if (n_cand > 0 && st->i_star < INT_MAX) {
            st->decided = 1; st->decided_entry = a.ent[st->i_star];
            if (!ARRAY) st->decided_call = st->calls;
        }
        FPResult r;
        r.decided = st->decided; r.received = st->votes_received; r.len = 0; r.count = 0; r.h1 = 0; r.h2 = 0;
        r.decided_call = st->decided_call; r.bad_sender = st->bad_sender;
        if (!ARRAY) st->calls = st->calls + 1;                // decided_call counts rapid_fp_tally_cd[_async] calls only
        if (r.decided && st->decided_entry >= 0) {
            const int32_t e = st->decided_entry;
            r.h1 = a.t_h1[e]; r.h2 = a.t_h2[e]; r.len = a.t_len[e]; r.count = *(volatile int32_t*)&a.t_count[e];
        }
        if (too_many) r.decided = -1;                        // reported as RAPID_EUNSUPPORTED by the host
        *a.out = r;
        st->n_call = 0; st->n_cand = 0; st->i_star = INT_MAX; st->bad_sender = -1; st->ticket = 0;
    }
}

static int32_t fp_reset_call_state(FP* fp) {        // per-call fields only; no host round trip
    k_fp_begin<<<1, 1, 0, fp->stream>>>(fp->st.p);
    RAPID_KERNEL_CHECK();
    return RAPID_OK;
}

// the grid of k_fp_tally (co-resident blocks of the smallest instantiation, so that any runs on it) and its scratch for R votes
static int32_t tally_reserve(FP* fp, int64_t R) {
    if (fp->tally_grid == 0) {
        int dev = 0, sms = TARGET_SMS, per_cd = 4, per_array = 4, per_wire = 4;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_cd, k_fp_tally<false>, TALLY_THREADS, 0);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_array, k_fp_tally<true>, TALLY_THREADS, 0);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_wire, k_fp_tally<true, true>, TALLY_THREADS, 0);
        fp->tally_grid = std::max(1, sms * std::max(std::min(std::min(per_cd, per_array), per_wire), 1));
        RAPID_CHECK(fp->blk_cnt.reserve((size_t)8 * fp->tally_grid));
    }
    return fp->ent.reserve((size_t)std::max<int64_t>(R, 1));
}

// launch k_fp_tally over ta.R votes (ta holds their source; tally_reserve(fp, ta.R) came first) on the tally's stream; the
// result record goes to d_res_raw
static int32_t tally_launch(FP* fp, TallyArgs& ta, bool array, bool wire = false) {
    ta.sender_cap = fp->sender_cap; ta.seen = fp->seen.p; ta.T = fp->T;
    ta.t_state = fp->t_state.p; ta.t_h1 = fp->t_h1.p; ta.t_h2 = fp->t_h2.p; ta.t_len = fp->t_len.p;
    ta.t_count = fp->t_count.p; ta.t_call = fp->t_call.p; ta.ent = fp->ent.p;
    ta.entries = fp->entries.p; ta.call_list = fp->call_list.p; ta.blk_cnt = fp->blk_cnt.p;
    ta.st = fp->st.p; ta.Q = (int32_t)fp->Q; ta.sumbuf = fp->sumbuf.p;
    ta.out = (FPResult*)fp->d_res_raw.p;
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(fp->tally_grid, ceil_div<int64_t>(ta.R, TALLY_THREADS)));
    void* args[] = {(void*)&ta};
    void* k = wire ? (void*)k_fp_tally<true, true> : array ? (void*)k_fp_tally<true> : (void*)k_fp_tally<false>;
    RAPID_CUDA(cudaLaunchCooperativeKernel(k, dim3((unsigned)grid),
                                           dim3(TALLY_THREADS), args, 0, fp->stream));
    fp->last_launches = 1;
    return RAPID_OK;
}

// the host copy of k_fp_tally's result record -> the caller's outputs, or the refusal it reports
static int32_t take_result(FP* fp, int32_t* decided, uint64_t* dh1, uint64_t* dh2, int32_t* dlen, int32_t* dcount, int32_t* received,
                           int32_t* decided_in_call, const int32_t* wire_sender = nullptr) {
    const FPResult r = *(const FPResult*)fp->h_res_raw.p;
    if (r.bad_sender >= 0) {
        if (wire_sender && *wire_sender < 0)
            set_error("vote %d of the current configuration comes from an endpoint outside the dictionary", r.bad_sender);
        else set_error("vote %d: sender id outside [0, sender_capacity)", r.bad_sender);
        return RAPID_EINVAL;
    }
    if (r.decided < 0) { set_error("more than 8 proposals reached the quorum in one call"); return RAPID_EUNSUPPORTED; }
    fp->decided_host = r.decided != 0;
    if (decided) *decided = r.decided;
    if (received) *received = r.received;
    if (dh1) *dh1 = r.h1;
    if (dh2) *dh2 = r.h2;
    if (dlen) *dlen = r.len;
    if (dcount) *dcount = r.count;
    if (decided_in_call) *decided_in_call = r.decided_call;
    return RAPID_OK;
}

}  // namespace rapid

using namespace rapid;

struct rapid_fp : rapid::FP {};

extern "C" {

int32_t rapid_fp_create(rapid_fp** out, int64_t cfg_id, int64_t membership_size, int64_t sender_capacity, int32_t device) {
    if (!out || membership_size < 1 || sender_capacity < 1 || sender_capacity > 0x7ffffff0LL) { set_error("bad arguments"); return RAPID_EINVAL; }
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); set_error("no CUDA device: librapid_b200 has no CPU fallback"); return RAPID_ECUDA; }
    if (device < 0 || device >= ndev) { set_error("device out of range"); return RAPID_EINVAL; }
    DeviceGuard g(device);
    rapid_fp* fp = new rapid_fp();
    fp->device = device;
    fp->cfg = cfg_id;
    fp->N = membership_size;
    fp->Q = membership_size - (membership_size - 1) / 4;            // FastPaxos.java:145
    fp->sender_cap = sender_capacity;
    uint32_t T = 1024;
    while ((int64_t)T < 2 * sender_capacity) T <<= 1;
    fp->T = T;
    int32_t rc = RAPID_OK;
    do {
        if (cudaStreamCreateWithFlags(&fp->stream, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreate(&fp->ev0) != cudaSuccess ||
            cudaEventCreate(&fp->ev1) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "stream", __FILE__, __LINE__); break; }
        if ((rc = fp->seen.reserve((size_t)sender_capacity))) break;
        if ((rc = fp->t_state.reserve(T))) break;
        if ((rc = fp->t_len.reserve(T))) break;
        if ((rc = fp->t_count.reserve(T))) break;
        if ((rc = fp->t_call.reserve(T))) break;
        if ((rc = fp->entries.reserve(T))) break;
        if ((rc = fp->call_list.reserve(T))) break;
        if ((rc = fp->t_h1.reserve(T))) break;
        if ((rc = fp->t_h2.reserve(T))) break;
        if ((rc = fp->st.reserve(1))) break;
        if ((rc = fp->h_st.reserve(1))) break;
        if ((rc = fp->hist.reserve(65536))) break;
        if ((rc = fp->mm.reserve(8))) break;
        if ((rc = fp->h_mm.reserve(8))) break;
        if ((rc = fp->d_res_raw.reserve(128))) break;
        if ((rc = fp->h_res_raw.reserve(128))) break;
        const int TB = 256;
        k_fp_fill<<<(unsigned)ceil_div<int64_t>(sender_capacity, TB), TB, 0, fp->stream>>>(fp->seen.p, sender_capacity, INT_MAX);
        cudaMemsetAsync(fp->t_state.p, 0, T * sizeof(int32_t), fp->stream);
        cudaMemsetAsync(fp->t_count.p, 0, T * sizeof(int32_t), fp->stream);
        cudaMemsetAsync(fp->t_call.p, 0, T * sizeof(int32_t), fp->stream);
        cudaMemsetAsync(fp->st.p, 0, sizeof(FPState), fp->stream);
        k_fp_reset<<<1, 32, 0, fp->stream>>>(0, fp->seen.p, 0, fp->t_state.p, fp->t_count.p, fp->t_call.p, fp->st.p);   // i_star = INT_MAX, bad_sender = -1
        if (cudaStreamSynchronize(fp->stream) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "init", __FILE__, __LINE__); break; }
    } while (0);
    if (rc) { rapid_fp_destroy(fp); return rc; }
    *out = fp;
    return RAPID_OK;
}

// A new FastPaxos instance for the next configuration (MembershipService.java:427-429) on the same buffers.
int32_t rapid_fp_reset(rapid_fp* fp, int64_t cfg_id, int64_t membership_size) {
    if (!fp || membership_size < 1) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(fp->device);
    cudaStream_t s = fp->stream;
    fp->cfg = cfg_id;
    fp->N = membership_size;
    fp->Q = membership_size - (membership_size - 1) / 4;
    fp->decided_host = false;
    const int TB = 256;
    const int64_t m = std::max<int64_t>(fp->sender_cap, (int64_t)fp->T);
    k_fp_reset<<<(unsigned)ceil_div<int64_t>(m, TB), TB, 0, s>>>(fp->sender_cap, fp->seen.p, fp->T, fp->t_state.p, fp->t_count.p, fp->t_call.p, fp->st.p);
    RAPID_KERNEL_CHECK();
    return RAPID_OK;      // asynchronous: everything that follows runs on the same stream
}

int32_t rapid_fp_destroy(rapid_fp* fp) {
    if (!fp) return RAPID_OK;
    DeviceGuard g(fp->device);
    if (fp->stream) cudaStreamSynchronize(fp->stream);
    if (fp->ev0) cudaEventDestroy(fp->ev0);
    if (fp->ev1) cudaEventDestroy(fp->ev1);
    if (fp->stream) cudaStreamDestroy(fp->stream);
    delete fp;
    return RAPID_OK;
}

int32_t rapid_fp_tally(rapid_fp* fp, int64_t n_votes, const int32_t* sender, const int64_t* vote_cfg, const uint64_t* proposal_hash,
                       const uint64_t* proposal_hash2, const int32_t* proposal_len, int32_t* decided, uint64_t* decided_hash,
                       uint64_t* decided_hash2, int32_t* decided_len, int32_t* decided_count, int32_t* votes_received) {
    if (!fp || n_votes < 0 || (n_votes && (!sender || !proposal_hash))) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(fp->device);
    cudaStream_t s = fp->stream;
    const int64_t n = fp->decided_host ? 0 : n_votes;      // :138 — everything after the decision is ignored
    const size_t m = (size_t)std::max<int64_t>(n, 1);
    RAPID_CHECK(fp->v_sender.reserve(m));
    RAPID_CHECK(fp->v_h1.reserve(m));
    RAPID_CHECK(tally_reserve(fp, n));
    RAPID_CUDA(cudaEventRecord(fp->ev0, s));
    if (n) {
        RAPID_CUDA(cudaMemcpyAsync(fp->v_sender.p, sender, (size_t)n * 4, cudaMemcpyHostToDevice, s));
        RAPID_CUDA(cudaMemcpyAsync(fp->v_h1.p, proposal_hash, (size_t)n * 8, cudaMemcpyHostToDevice, s));
        if (vote_cfg) { RAPID_CHECK(fp->v_cfg.reserve(m)); RAPID_CUDA(cudaMemcpyAsync(fp->v_cfg.p, vote_cfg, (size_t)n * 8, cudaMemcpyHostToDevice, s)); }
        if (proposal_hash2) { RAPID_CHECK(fp->v_h2.reserve(m)); RAPID_CUDA(cudaMemcpyAsync(fp->v_h2.p, proposal_hash2, (size_t)n * 8, cudaMemcpyHostToDevice, s)); }
        if (proposal_len) { RAPID_CHECK(fp->v_len.reserve(m)); RAPID_CUDA(cudaMemcpyAsync(fp->v_len.p, proposal_len, (size_t)n * 4, cudaMemcpyHostToDevice, s)); }
    }
    TallyArgs ta = {};
    ta.R = n; ta.sender = fp->v_sender.p; ta.vcfg = vote_cfg ? fp->v_cfg.p : nullptr; ta.cfg = fp->cfg;
    ta.h1v = fp->v_h1.p; ta.h2v = proposal_hash2 ? fp->v_h2.p : nullptr; ta.lenv = proposal_len ? fp->v_len.p : nullptr;
    RAPID_CHECK(tally_launch(fp, ta, true));
    RAPID_CUDA(cudaEventRecord(fp->ev1, s));
    RAPID_CUDA(cudaMemcpyAsync(fp->h_res_raw.p, fp->d_res_raw.p, sizeof(FPResult), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    cudaEventElapsedTime(&fp->last_ms, fp->ev0, fp->ev1);
    return take_result(fp, decided, decided_hash, decided_hash2, decided_len, decided_count, votes_received, nullptr);
}

int32_t rapid_fp_tally_wire(rapid_fp* fp, const rapid_wire* w, int32_t* decided, uint64_t* decided_hash, uint64_t* decided_hash2,
                            int32_t* decided_len, int32_t* decided_count, int32_t* votes_received) {
    if (!fp) { set_error("NULL handle"); return RAPID_EINVAL; }
    WireMsgs m;
    RAPID_CHECK(wire_consensus_dev(w, RAPID_WIRE_FAST_ROUND_PHASE2B, &m));
    if (m.device != fp->device) { set_error("fp and wire live on different devices"); return RAPID_EINVAL; }
    DeviceGuard g(fp->device);
    cudaStream_t s = fp->stream;
    const int64_t n = fp->decided_host ? 0 : m.n;          // :138 — everything after the decision is ignored
    RAPID_CHECK(tally_reserve(fp, n));
    RAPID_CUDA(cudaEventRecord(fp->ev0, s));
    TallyArgs ta = {};
    ta.R = n; ta.sender = m.sender; ta.vcfg = m.cfg; ta.cfg = fp->cfg; ta.h1v = m.h1; ta.h2v = m.h2; ta.lenv = m.len;
    RAPID_CHECK(tally_launch(fp, ta, true, true));
    RAPID_CUDA(cudaEventRecord(fp->ev1, s));
    RAPID_CUDA(cudaMemcpyAsync(fp->h_res_raw.p, fp->d_res_raw.p, sizeof(FPResult), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    cudaEventElapsedTime(&fp->last_ms, fp->ev0, fp->ev1);
    int32_t bad = 0;                                        // the refused vote's sender: -1 (unknown endpoint) or past sender_capacity
    const FPResult r = *(const FPResult*)fp->h_res_raw.p;
    if (r.bad_sender >= 0) RAPID_CUDA(cudaMemcpy(&bad, m.sender + r.bad_sender, 4, cudaMemcpyDeviceToHost));
    return take_result(fp, decided, decided_hash, decided_hash2, decided_len, decided_count, votes_received, nullptr, &bad);
}

// enqueue the tally of the detector's votes (and, sharded, the all-reduce + decision kernel) on the tally's stream
static int32_t tally_cd_enqueue(rapid_fp* fp, const rapid_cd* cd, rapid_comm* comm) {
    if (!fp || !cd) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (fp->device != cd->device) { set_error("fp and cd live on different devices"); return RAPID_EINVAL; }
    if (cd->raw) { set_error("RAW detectors do not announce proposals"); return RAPID_EINVAL; }
    if (comm && comm->device != fp->device) { set_error("comm and fp live on different devices"); return RAPID_EINVAL; }
    cudaStream_t s = fp->stream;
    RAPID_CHECK(tally_reserve(fp, cd->R));
    // The detector's outputs are produced on ITS stream (possibly by an asynchronous batch still in flight): order this
    // tally after them on the device instead of waiting on the host.
    RAPID_CUDA(cudaStreamWaitEvent(s, cd->ev_done, 0));
    RAPID_CUDA(cudaEventRecord(fp->ev0, s));
    const bool direct = comm != nullptr;
    const size_t words = (size_t)(SUM_BUCKETS + 1) * SUM_WORDS;
    if (direct) {
        RAPID_CHECK(fp->sumbuf.reserve(words));
        RAPID_CUDA(cudaMemsetAsync(fp->sumbuf.p, 0, words * sizeof(unsigned long long), s));
    }
    TallyArgs ta = {};
    ta.R = cd->R; ta.rbegin = cd->rbegin; ta.rflags = cd->rflags.p; ta.ring0 = cd->view->ring.p;
    ta.h1v = cd->out_h1.p; ta.h2v = cd->out_h2.p; ta.lenv = cd->out_len.p;
    ta.direct = direct ? 1 : 0;
    RAPID_CHECK(tally_launch(fp, ta, false));
    fp->pending_comm = comm;
    fp->pending_cd = cd;
    if (direct && getenv("RAPID_B200_FORCE_REFINE") == nullptr) {
        // sharded: count-weighted sums of the local table -> ONE all-reduce (sum) -> the winning bucket gives the proposal back
        // by exact division (RAPID_B200_FORCE_REFINE: test hook that skips this and takes the digit-by-digit refinement)
        RAPID_NCCL(g_nccl.AllReduce(fp->sumbuf.p, fp->sumbuf.p, words, NCCL_UINT64, NCCL_SUM, comm->comm, s));
        k_fp_decide_sum<<<1, 1024, 0, s>>>(fp->sumbuf.p, (unsigned long long)fp->Q, (FPSumResult*)fp->d_res_raw.p, fp->st.p);
        RAPID_KERNEL_CHECK();
        fp->last_launches += 1;
    }
    RAPID_CUDA(cudaMemcpyAsync(fp->h_res_raw.p, fp->d_res_raw.p, sizeof(FPSumResult), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaEventRecord(fp->ev1, s));
    return RAPID_OK;
}

static int32_t tally_cd_refine(rapid_fp* fp, rapid_comm* comm, int32_t* decided, uint64_t* decided_hash, uint64_t* decided_hash2,
                               int32_t* decided_len, int32_t* decided_count, int32_t* votes_received);

// wait for the last enqueued tally and read its outcome (ONE host synchronisation)
static int32_t tally_cd_collect(rapid_fp* fp, int32_t* decided, uint64_t* decided_hash, uint64_t* decided_hash2, int32_t* decided_len,
                                int32_t* decided_count, int32_t* votes_received, int32_t* decided_in_call) {
    cudaStream_t s = fp->stream;
    RAPID_CUDA(cudaStreamSynchronize(s));
    cudaEventElapsedTime(&fp->last_ms, fp->ev0, fp->ev1);
    cudaGetLastError();
    if (fp->pending_cd) RAPID_CHECK(cd_wait(fp->pending_cd, true));      // outcome of the (asynchronous) batches these votes came from
    rapid_comm* comm = fp->pending_comm;
    if (comm == nullptr)
        return take_result(fp, decided, decided_hash, decided_hash2, decided_len, decided_count, votes_received, decided_in_call);
    if (getenv("RAPID_B200_FORCE_REFINE") == nullptr) {              // (test hook, see above)
        const FPSumResult res = *(const FPSumResult*)fp->h_res_raw.p;
        if (!res.ambiguous) {
            if (res.r.decided) fp->decided_host = true;
            if (decided) *decided = res.r.decided;
            if (decided_hash) *decided_hash = res.r.h1;
            if (decided_hash2) *decided_hash2 = res.r.h2;
            if (decided_len) *decided_len = res.r.len;
            if (decided_count) *decided_count = res.r.count;
            if (votes_received) *votes_received = res.r.received;
            if (decided_in_call) *decided_in_call = res.r.decided_call;
            return RAPID_OK;
        }
        // two proposals share a quorum-sized bucket (every rank sees the same flag): digit-by-digit refinement
    }
    if (decided_in_call) *decided_in_call = -1;
    return tally_cd_refine(fp, comm, decided, decided_hash, decided_hash2, decided_len, decided_count, votes_received);
}

int32_t rapid_fp_tally_cd(rapid_fp* fp, const rapid_cd* cd, rapid_comm* comm, int32_t* decided, uint64_t* decided_hash,
                          uint64_t* decided_hash2, int32_t* decided_len, int32_t* decided_count, int32_t* votes_received) {
    if (!fp) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(fp->device);
    RAPID_CHECK(tally_cd_enqueue(fp, cd, comm));
    return tally_cd_collect(fp, decided, decided_hash, decided_hash2, decided_len, decided_count, votes_received, nullptr);
}

int32_t rapid_fp_tally_cd_async(rapid_fp* fp, const rapid_cd* cd, rapid_comm* comm) {
    if (!fp) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(fp->device);
    return tally_cd_enqueue(fp, cd, comm);
}

// One configuration epoch of a virtual cluster, enqueued in ONE call: clear() of the detectors + a new FastPaxos instance
// (decideViewChange's resets, MembershipService.java:425-429), one alert batch resident on the device, and the fast-round tally of
// the proposals it produces — nothing waits on the host; rapid_fp_result collects the decision.
int32_t rapid_fp_epoch_async(rapid_fp* fp, rapid_cd* cd, rapid_comm* comm, int64_t cfg_id, int64_t membership_size, int64_t n_cells,
                             const int32_t* dst_dev, const uint8_t* ring_dev, const uint8_t* status_dev, const int64_t* cell_cfg_dev,
                             const rapid_delivery* delivery_dev) {
    RAPID_CHECK(rapid_cd_clear(cd));
    RAPID_CHECK(rapid_fp_reset(fp, cfg_id, membership_size));
    RAPID_CHECK(rapid_cd_apply_batch_dev_async(cd, cfg_id, n_cells, nullptr, dst_dev, ring_dev, status_dev, cell_cfg_dev, delivery_dev));
    return rapid_fp_tally_cd_async(fp, cd, comm);
}

int32_t rapid_fp_result(rapid_fp* fp, int32_t* decided, uint64_t* decided_hash, uint64_t* decided_hash2, int32_t* decided_len,
                        int32_t* decided_count, int32_t* votes_received, int32_t* decided_in_call) {
    if (!fp) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (!fp->pending_cd) { set_error("no rapid_fp_tally_cd_async call to collect"); return RAPID_EINVAL; }
    DeviceGuard g(fp->device);
    return tally_cd_collect(fp, decided, decided_hash, decided_hash2, decided_len, decided_count, votes_received, decided_in_call);
}

// the rare path: a quorum-sized bucket of the sum buffer holds more than one fingerprint
static int32_t tally_cd_refine(rapid_fp* fp, rapid_comm* comm, int32_t* decided, uint64_t* decided_hash, uint64_t* decided_hash2,
                               int32_t* decided_len, int32_t* decided_count, int32_t* votes_received) {
    cudaStream_t s = fp->stream;
    const int TB = 256;
    const unsigned gt = (unsigned)ceil_div<uint32_t>(fp->T, TB);
    RAPID_CUDA(cudaEventRecord(fp->ev0, s));
    RAPID_CUDA(cudaMemcpyAsync(fp->h_st.p, fp->st.p, sizeof(FPState), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    Prefix pf;
    pf.n = 0;
    int32_t dec = 0, dcount = 0, dlen = 0;
    uint64_t dh1 = 0, dh2 = 0;
    for (int level = 0; level < 8 && !dec; ++level) {
        RAPID_CUDA(cudaMemsetAsync(fp->hist.p, 0, 65536 * sizeof(int32_t), s));
        k_fp_hist<<<gt, TB, 0, s>>>(fp->T, fp->t_state.p, fp->t_h1.p, fp->t_h2.p, fp->t_count.p, pf, fp->hist.p);
        RAPID_KERNEL_CHECK();
        RAPID_NCCL(g_nccl.AllReduce(fp->hist.p, fp->hist.p, 65536, NCCL_INT32, NCCL_SUM, comm->comm, s));
        RAPID_CHECK(fp_reset_call_state(fp));
        k_fp_hist_cand<<<65536 / TB, TB, 0, s>>>(fp->hist.p, (int32_t)fp->Q, fp->st.p);
        RAPID_KERNEL_CHECK();
        fp->last_launches += 2;
        RAPID_CUDA(cudaMemcpyAsync(fp->h_st.p, fp->st.p, sizeof(FPState), cudaMemcpyDeviceToHost, s));
        RAPID_CUDA(cudaStreamSynchronize(s));
        const FPState st = *fp->h_st.p;
        if (st.n_cand == 0) break;                                   // nothing reaches the quorum
        // senders are members here, so at most one proposal can reach Q > N/2: follow the first candidate bucket
        pf.d[pf.n++] = (uint32_t)st.cand[0];
        int32_t bucket_count = 0;
        RAPID_CUDA(cudaMemcpyAsync(&bucket_count, fp->hist.p + st.cand[0], 4, cudaMemcpyDeviceToHost, s));
        RAPID_CUDA(cudaMemsetAsync(fp->mm.p, 0, 8 * sizeof(unsigned long long), s));
        k_fp_minmax<<<gt, TB, 0, s>>>(fp->T, fp->t_state.p, fp->t_h1.p, fp->t_h2.p, fp->t_len.p, fp->t_count.p, pf, fp->mm.p);
        RAPID_KERNEL_CHECK();
        fp->last_launches += 1;
        RAPID_NCCL(g_nccl.AllReduce(fp->mm.p, fp->mm.p, 6, NCCL_UINT64, NCCL_MAX, comm->comm, s));
        RAPID_CUDA(cudaMemcpyAsync(fp->h_mm.p, fp->mm.p, 6 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
        RAPID_CUDA(cudaStreamSynchronize(s));
        const unsigned long long* mm = fp->h_mm.p;
        if (mm[0] == ~mm[1] && mm[2] == ~mm[3] && mm[4] == ~mm[5]) {  // one fingerprint in the bucket: its count is exact
            dec = 1; dcount = bucket_count; dh1 = mm[0]; dh2 = mm[2]; dlen = (int32_t)mm[4];
        }
    }
    int32_t recv_local = fp->h_st.p->votes_received, recv = 0;
    {   // votesReceived across ranks (tiny all-reduce on the same stream)
        RAPID_CUDA(cudaMemsetAsync(fp->hist.p, 0, sizeof(int32_t), s));
        RAPID_CUDA(cudaMemcpyAsync(fp->hist.p, &recv_local, 4, cudaMemcpyHostToDevice, s));
        RAPID_NCCL(g_nccl.AllReduce(fp->hist.p, fp->hist.p, 1, NCCL_INT32, NCCL_SUM, comm->comm, s));
        RAPID_CUDA(cudaMemcpyAsync(&recv, fp->hist.p, 4, cudaMemcpyDeviceToHost, s));
    }
    RAPID_CUDA(cudaEventRecord(fp->ev1, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    cudaEventElapsedTime(&fp->last_ms, fp->ev0, fp->ev1);
    if (dec) {      // remember the decision locally so later votes are ignored (:138)
        FPState stn = *fp->h_st.p;
        stn.decided = 1; stn.decided_entry = -1;
        *fp->h_st.p = stn;
        RAPID_CUDA(cudaMemcpy(fp->st.p, fp->h_st.p, sizeof(FPState), cudaMemcpyHostToDevice));
        fp->decided_host = true;
    }
    if (decided) *decided = dec;
    if (decided_hash) *decided_hash = dh1;
    if (decided_hash2) *decided_hash2 = dh2;
    if (decided_len) *decided_len = dlen;
    if (decided_count) *decided_count = dcount;
    if (votes_received) *votes_received = recv;
    return RAPID_OK;
}

int32_t rapid_fp_timer_stop(rapid_fp* fp, const rapid_cd* cd, float* out_ms) {
    if (!fp || !cd || !out_ms) { set_error("NULL argument"); return RAPID_EINVAL; }
    if (fp->device != cd->device) { set_error("fp and cd live on different devices"); return RAPID_EINVAL; }
    DeviceGuard g(fp->device);
    RAPID_CUDA(cudaStreamWaitEvent(fp->stream, cd->ev_done, 0));
    RAPID_CUDA(cudaEventRecord(fp->ev1, fp->stream));
    RAPID_CUDA(cudaStreamSynchronize(fp->stream));
    RAPID_CHECK(cd_wait(cd, false));
    RAPID_CUDA(cudaEventElapsedTime(out_ms, cd->ev_t0, fp->ev1));
    return RAPID_OK;
}

int32_t rapid_fp_last_device_ms(const rapid_fp* fp, float* total_ms) {
    if (!fp) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (total_ms) *total_ms = fp->last_ms;
    return RAPID_OK;
}

int32_t rapid_fp_last_launches(const rapid_fp* fp, int32_t* n_kernel_launches) {
    if (!fp || !n_kernel_launches) { set_error("NULL argument"); return RAPID_EINVAL; }
    *n_kernel_launches = fp->last_launches;
    return RAPID_OK;
}

int32_t rapid_comm_unique_id(void* out_id) {
    if (!out_id) { set_error("NULL argument"); return RAPID_EINVAL; }
    RAPID_CHECK(load_nccl());
    nccl_uid id;
    RAPID_NCCL(g_nccl.GetUniqueId(&id));
    memcpy(out_id, &id, sizeof(id));
    return RAPID_OK;
}

int32_t rapid_comm_init(rapid_comm** out, int32_t rank, int32_t world, const void* nccl_unique_id, int32_t device) {
    if (!out || !nccl_unique_id || world < 1 || rank < 0 || rank >= world) { set_error("bad arguments"); return RAPID_EINVAL; }
    *out = nullptr;
    RAPID_CHECK(load_nccl());
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) { cudaGetLastError(); set_error("bad device"); return RAPID_ECUDA; }
    RAPID_CUDA(cudaSetDevice(device));
    rapid_comm* c = new rapid_comm();
    c->device = device; c->rank = rank; c->world = world;
    nccl_uid id;
    memcpy(&id, nccl_unique_id, sizeof(id));
    int r = g_nccl.CommInitRank(&c->comm, world, id, rank);
    if (r != 0) { set_error("ncclCommInitRank failed: %d (%s)", r, g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"); delete c; return RAPID_ENCCL; }
    *out = c;
    return RAPID_OK;
}

int32_t rapid_comm_destroy(rapid_comm* c) {
    if (!c) return RAPID_OK;
    if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
    delete c;
    return RAPID_OK;
}

}  // extern "C"
