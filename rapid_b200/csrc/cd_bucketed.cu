// The subject-bucketed cut-detection kernels (the fast path of rapid_cd_apply_batch on SERVICE handles).
//
// Reference semantics: MultiNodeCutDetector.java:84-128 applied per cell in arrival order, then :137-164, driven
// by MembershipService.java:300-354.  The Java walks the batch once per process and probes a hash map per cell.
// Here the batch is regrouped BY SUBJECT once (counting sort by subject slot inside cd_prepare.cu), and every receiver's
// state word for a subject (10 ring bits at K <= 10, see RowRef) is read ONCE, updated in a register and written ONCE:
//
//   traffic = 2.5 bytes x (#subjects in the batch) x (#receivers)        (SURVEY.md §8d "4·S·R" with 16-bit words)
//
// instead of 4 bytes x #cells x #receivers for a per-cell sweep.  What makes that legal is that the sequential
// rule "emit when updatesInProgress returns to 0" only depends on, per subject, the two moments at which its
// report count crosses L and H (t_L, t_H): a proposal is emitted at t_H(s) iff no other subject s' has
// t_L(s') <= t_H(s) < t_H(s') (SURVEY.md §7 "key reformulation").  Each (subject, receiver) visit yields
// (t_L, t_H); per receiver we keep a handful of order-independent reductions of them and classify:
//     all pre-proposals resolved  -> everything at >= H is emitted              (EMIT_ALL)
//     an unresolved one starts before the first H-crossing -> nothing emitted   (NOEMIT)
//     otherwise                                                                  (MIXED: exact interval analysis
//                                                                                 for that receiver only)
// followed by the implicit-invalidation pass over the (few) subjects left in the unstable band.
//
// "Moments" are cell indices for uniform delivery and the receiver's own permutation keys for PERMUTED delivery,
// so a per-receiver order needs no per-receiver sort.
//
// A batch is a fixed chain of launches with no host round trip between them (cd_prepare.cu's k_prepare, then the kernels below); the
// host learns the outcome from a snapshot of the device counters at its next synchronisation point:
//   k_apply_uniform<PERM, SEQ, HB>  SWAR, 8 receivers per thread, lo + hi plane group loads/stores, write-only fresh-subject path, per-block memo +
//                          L2 prefetch on the read-modify-write path.  PERM = every receiver gets every cell but in its OWN order
//                          (RAPID_DELIVERY_PERMUTED): the new state and all the crossing COUNTS do not depend on the order, so the
//                          kernel is the uniform one minus the moments; the (rare) receivers whose classification needs their own
//                          t_L / t_H get them from a per-receiver pass over the pre-batch rows inside k_mixed_flip.  SEQ = a sequence
//                          of batches in one pass (rapid_cd_apply_batches), checked per receiver by k_seq_check.
//   k_apply_generic        one receiver per thread: per-receiver delivery bitmaps (with or without a permuted order)
//   k_finalize1            classification per receiver (EMIT_ALL / NOEMIT / MIXED) from the partial accumulators
//   k_mixed_flip           cooperative, always launched: [moments on demand] -> [interval analysis to its fixpoint] -> row flip
//   k_inval_finalize2      invalidateFailingEdges over the work list + the receivers' closing bookkeeping
//   k_marks                cooperative, returns at once unless some receiver went through the interval analysis: emit marks,
//                          counter snapshot
#include <cooperative_groups.h>

#include <algorithm>
#include <climits>
#include <cstdlib>

#include "cd_internal.cuh"

namespace cg = cooperative_groups;

namespace rapid {

// Tuning choices (why each was made: DESIGN.md §4.2 and §4.3):
// k_apply_uniform: resident blocks/SM its register budget is sized for.  5 = 96 registers; at 8 (64) every instantiation spills
// on sm_90a and the kernel is slower (A/B in DESIGN.md §4.2).
constexpr int UNI_MINBLOCKS = 5;
// k_apply_uniform, carried subjects: the rows of the next PF_DIST staged subjects are prefetched into L2 (DESIGN.md §4.2).
constexpr int PF_DIST = 2;
// k_apply_uniform, carried subjects: the visit of the tile's sample state is computed once per block (memo, DESIGN.md §4.2).
// k_inval_finalize2: below 64 tiles a tile's work list is split over several blocks (DESIGN.md §4.3).

constexpr int TILE_R = 1024;          // receivers per tile (uniform kernel: 128 threads x 8 receivers)
constexpr int UNI_THREADS = 128;
constexpr int GEN_THREADS = 256;
constexpr int STAGE = 32;             // batch subjects staged in shared memory at a time
constexpr int MAXK = RAPID_MAX_K;
constexpr int SMALL_SEG = 4;          // generic visit: subjects with at most this many cells in the batch stay in registers
constexpr uint32_t T32_NONE = 0xFFFFFFFFu;
constexpr uint64_t T64_NONE = ~0ULL;
constexpr uint32_t RF_K3 = 16u;       // receiver enters the invalidation pass of the batch in flight
constexpr uint32_t RF_ACTIVE = 32u;   // receiver processed the batch in flight
constexpr uint32_t RF_MIXED_EMIT = 64u;   // announced a proposal found by the interval analysis: "emitted" == t_H <= estar[r]

// per-receiver state of the interval analysis (MIXED receivers)
constexpr uint32_t MX_ON = 1u, MX_NEG = 2u, MX_HAS_E = 4u, MX_DONE = 8u;
constexpr uint32_t MX_REF = 32u;      // resolved through the reference receiver (its sums are already in mx_e1 / mx_e2 / mx_ec)
constexpr uint32_t MX_TIME = 16u;     // PERMUTED delivery: the classification needs this receiver's own min t_H / min t_L

// partial-accumulator flags
constexpr uint32_t PF_SEEN = 1u;      // a valid DOWN cell was delivered
constexpr uint32_t PF_NEGINF = 2u;    // a subject already in the unstable band stayed there (its t_L is "before the batch")

// Counts are full 32-bit words wherever they sum over more than one stage of subjects: a chunk (or a whole batch) can hold
// 65,536 subjects or more.  The 16-bit halves of StageAcc only ever hold the sum over one stage (at most STAGE subjects).
struct ChunkAcc {                     // what the FRESH subjects of a chunk contribute to EVERY active receiver
    uint32_t nL, nH, tp, nUn, fl, minTH, minTLun, pad_;
    uint64_t h1, h2;
    // sequences of batches: the prefix part (batches before the last one)
    uint32_t nLp, nHp, tpc, minBHp, minBLlong, pad2_;
    uint64_t h1p, h2p;
};

// Partials::cnt.z holds touched_pre in its low 30 bits and the PF_* flags above them: a chunk holds fewer than 2^30 subjects
// (the slot count is bounded far below that by the state rows, at least 3 * Rpad bytes per slot)
constexpr int PF_SHIFT = 30;
constexpr uint32_t TP_MASK = (1u << PF_SHIFT) - 1u;

struct Partials {                     // [n_chunks][Rpad] structure of arrays
    uint4* cnt;                       // x = nL, y = nH, z = touched_pre | flags << PF_SHIFT, w = nUn
    uint4* cntp;                      // sequences only: x = nLp, y = nHp, z = tpc (touched and in the band before the call)
    uint64_t* minTH;
    uint64_t* minTLun;
    uint64_t* h1;
    uint64_t* h2;
    uint64_t* h1p;                    // sequences only: fingerprint of the subjects that reached H in the prefix
    uint64_t* h2p;
    uint2* seq;                       // sequences only: x = min prefix batch with an H-crossing, y = min L-batch of a subject still in
                                      // the band when the last batch starts (0 = since before the call)
    int32_t* flag;                    // [n_chunks][n_tiles] 1 = the per-receiver partials of this (chunk, tile) were written
    ChunkAcc* chunk;                  // [n_chunks] used for (chunk, tile) pairs whose flag is 0
    int n_tiles;
};

struct Bucketed {
    DevBuf<int32_t> sidx;                     // cell indices grouped by subject (arrival order inside a subject)
    DevBuf<int32_t> seg_cnt, batch_slots;     // [slot] scratch of the prepare kernel (seg_cnt all zero between batches)
    DevBuf<int32_t> bins, ovf, cell_batch;    // [slot][64] cell bins (PREP_BIN), [A] overflow list, [A] batch of every cell (sequences)
    DevBuf<SubjDesc> desc;
    DevBuf<SubjWalk> walk;
    DevBuf<uint8_t> s_ring, s_status;         // per sorted cell
    DevBuf<int32_t> p_flag;
    DevBuf<ChunkAcc> p_chunk;
    DevBuf<uint4> p_cnt, p_cntp;
    DevBuf<uint64_t> p_minTH, p_minTLun, p_h1, p_h2, p_h1p, p_h2p;
    DevBuf<uint2> p_seq;
    DevBuf<SubjWalk> pwalk;                   // sequences: prefix walks
    DevBuf<unsigned char> ra_dev;             // the ResolveArgs of the batch in flight (the kernels take a pointer: the struct is
                                              // too big to pass by value to the out-of-line rare paths without a per-thread copy)
    DevBuf<uint32_t> mx_fl;                   // [Rpad] MX_* flags
    DevBuf<uint64_t> mx_a, mx_cand, mx_emax;  // [Rpad] start of the never-closing component / its next candidate / e* candidate
    DevBuf<uint64_t> mx_p1, mx_p2;            // [Rpad] fingerprint of `proposal` before the batch
    DevBuf<int32_t> mx_pc;
    DevBuf<unsigned long long> mx_e1, mx_e2;  // [Rpad] fingerprint of the batch subjects emitted explicitly
    DevBuf<int32_t> mx_ec;
    DevBuf<uint64_t> estar;                   // [Rpad] last explicit emission moment of RF_MIXED_EMIT receivers
    DevBuf<int32_t> mx_changed;               // [4] rotating "the component grew" counters of the fixpoint loop
    DevBuf<uint32_t> mx_dev;                  // [Rpad / 32]
    DevBuf<int32_t> batch_index;              // [slot] -> index of the subject in the batch in flight
    DevBuf<int32_t> inv_res, inv_ticket;      // [Rpad] / [n_tiles] hand-over of k_inval_finalize2's blocks (all zero between launches)
    DevBuf<unsigned long long> inv_h1, inv_h2;
    // invalidation work list (WorkList)
    DevBuf<int32_t> wl_slots, wl_count, wl_listed, wl_so_tab;
    DevBuf<uint8_t> wl_in_tile;               // [slot][n_tiles]
    DevBuf<uint8_t> has_so;                   // [slot] some observer of the subject has a slot (can get implicit reports)
    size_t in_list_slots = 0;                 // slots the work-list arrays are sized for
    int n_tiles = 0;
    size_t part_cap = 0;
    int slots_uniform = 0, slots_generic = 0;   // resident blocks of the apply kernels on this device
    int resolve_grid = 0;                       // co-resident blocks of the cooperative resolve kernel
};

// ------------------------------------------------------------------------------------------------------------------
// the (subject, receiver) visit, uniform delivery: old 16-bit state -> crossings and moments
// ------------------------------------------------------------------------------------------------------------------
struct Visit {
    int c0, c1;
    bool crossL, crossH;
    uint32_t tL, tH;
};

// `ur` is the receiver's state for the subject when the (last) batch starts: its stored word, plus — in a sequence of batches —
// the rings of the prefix (SubjDesc::pmask)
__device__ __forceinline__ Visit visit_uniform(uint32_t ur, const SubjDesc& d, const SubjWalk& w, int L, int H) {
    Visit v;
    v.tL = 0; v.tH = 0;
    if (ur == d.pmask) {                                // fresh subject: the descriptor already knows the answer
        v.c0 = __popc(ur); v.c1 = __popc(ur | d.bmask);
        v.tL = d.tLf; v.tH = d.tHf;
    } else {
        int c = __popc(ur);
        v.c0 = c;
        const int nr = d.nr;
        for (int q = 0; q < nr; ++q) {
            const int k = w.ring[q];
            const bool isnew = !((ur >> k) & 1u);
            c += isnew;
            if (isnew && c == L) v.tL = w.time[q];
            if (isnew && c == H) v.tH = w.time[q];
        }
        v.c1 = c;
    }
    v.crossL = v.c0 < L && v.c1 >= L;
    v.crossH = v.c0 < H && v.c1 >= H;
    return v;
}

// PERMUTED delivery (every cell reaches every active receiver, each in its own order): the counts before / after the batch
// do not depend on the order; the moments are left out (they are computed on demand, k_resolve's moment pass)
__device__ __forceinline__ Visit visit_counts(uint32_t ur, const SubjDesc& d, uint32_t RM, int L, int H) {
    Visit v;
    v.tL = 0; v.tH = 0;
    v.c0 = __popc(ur);
    v.c1 = __popc((ur | d.bmask) & RM);
    v.crossL = v.c0 < L && v.c1 >= L;
    v.crossH = v.c0 < H && v.c1 >= H;
    return v;
}

struct Acc {
    uint32_t nL = 0, nH = 0, tp = 0, nUn = 0, flags = 0;
    uint32_t minTH = T32_NONE, minTLun = T32_NONE;
    uint64_t h1 = 0, h2 = 0;
    // sequences of batches (SEQ kernels only): what the prefix did
    uint32_t nLp = 0, nHp = 0, tpc = 0, minBHp = T32_NONE, minBLlong = T32_NONE;
    uint64_t h1p = 0, h2p = 0;
};

__device__ __forceinline__ bool accumulate(Acc& a, const Visit& v, const SubjDesc& d, int L, int H) {
    if (v.c0 >= L && v.c0 < H) a.tp++;
    if (v.crossL) a.nL++;
    if (v.crossH) { a.nH++; a.minTH = min(a.minTH, v.tH); a.h1 += d.mix1; a.h2 += d.mix2; }
    if (v.c1 >= L && v.c1 < H) {                        // still in the unstable band after the batch
        if (v.crossL) { a.nUn++; a.minTLun = min(a.minTLun, v.tL); }
        else a.flags |= PF_NEGINF;
        return true;
    }
    return false;
}

// ---- sequences of batches in ONE pass ------------------------------------------------------------------------------------
// rapid_cd_apply_batches on a bucketed handle: B BatchedAlertMessages, handleMessage (MembershipService.java:300-354) once per
// batch in order — cells, invalidateFailingEdges, and the announcedProposal gating between batches.  If no receiver emits a
// proposal before the LAST batch and no invalidation pass at the end of an earlier batch adds a report, then the earlier batches
// (the "prefix") did nothing but set ring bits and move subjects across L / H — order-independent — and the whole call equals
// ONE batch (the last) applied to the state `stored word | prefix rings`.  That is what the SEQ kernels compute: one pass over the
// rows for the whole sequence instead of one per batch.  Both premises are CHECKED per receiver on the device (k_seq_check), with
// batch-granular sufficient conditions:
//   A1  no emission in the prefix: no H-crossing in the prefix at all, or a subject that is in the unstable band from a batch
//       strictly before the first H-crossing until the last batch starts (updatesInProgress never returns to 0 in between)
//   A2  no implicit report at the end of a prefix batch: for every (subject s, ring k, observer o) with both in the dictionary,
//       the first batch end at which s is in the band, o is in proposal U preProposal and a DOWN alert has been seen comes
//       after s reached H or ring k was reported anyway — or is not in the prefix
// A receiver that fails either test aborts the pass for EVERYONE before anything is committed (rows are double-buffered, the
// scalars are written by the finalize kernels): the host then replays the sequence batch by batch.
// One (subject, receiver) through the prefix.  `u[k]` (for the rings in `umask`) is the first prefix batch END (1-based) at which the
// subject's ring-k observer is in proposal U preProposal and a DOWN alert has been seen — from then on an invalidation pass reports
// ring k implicitly while the subject sits in the unstable band (MultiNodeCutDetector.java:147-158).  The walk merges the explicit
// first reports (during batch t) with those passes (at the END of batch e; a pass applies ALL its eligible rings, :151-157, even
// past H) in batch order.  Returns the state when the last batch starts; acc (may be null) receives the prefix's crossings.
__device__ __forceinline__ uint32_t prefix_core(Acc* acc, uint32_t ur, const SubjDesc& d, const SubjWalk& pw, const uint32_t* u,
                                                uint32_t umask, int L, int H, uint32_t last) {
    const int c0 = __popc(ur);
    int c = c0;
    uint32_t word = ur, bLp = 0, bHp = 0;
    if (ur == 0 && umask == 0) {                         // fresh subject without dictionary observers: the descriptor knows
        c = __popc(d.pmask); bLp = d.f_bLp; bHp = d.f_bHp; word = d.pmask;
    } else {
        const int np = __popc(d.pmask);
        uint32_t imp = umask & ~ur;                      // implicit candidates still open
        uint32_t bL = c >= L ? 0u : T32_NONE;
        int q = 0;
        for (;;) {
            while (q < np && ((word >> pw.ring[q]) & 1u)) ++q;                     // explicit entries already reported
            const uint32_t te = q < np ? pw.time[q] : T32_NONE;
            uint32_t ti = T32_NONE;
            if (imp && c >= L && c < H) {
                for (uint32_t m = imp; m; m &= m - 1) { const int k = __ffs(m) - 1; if (u[k] != T32_NONE) ti = min(ti, max(u[k], bL)); }
                if (ti > last) ti = T32_NONE;
            }
            if (ti != T32_NONE && ti < te) {             // the invalidation pass at the end of batch ti comes first
                for (uint32_t m = imp; m; m &= m - 1) {
                    const int k = __ffs(m) - 1;
                    if (u[k] == T32_NONE || u[k] > ti) continue;
                    word |= 1u << k; imp &= ~(1u << k);
                    ++c;
                    if (c == H) bHp = ti;
                }
                if (c >= H) imp = 0;                     // out of preProposal: no later pass touches it
            } else if (te != T32_NONE) {
                const int k = pw.ring[q];
                word |= 1u << k; imp &= ~(1u << k);
                ++c; ++q;
                if (c == L) { bL = te; bLp = te; }
                if (c == H) bHp = te;
            } else {
                break;
            }
        }
    }
    if (acc) {
        if (c0 >= L && c0 < H) acc->tpc++;               // in the band before the call, touched by the call
        if (c0 < L && c >= L) acc->nLp++;
        if (c0 < H && c >= H) { acc->nHp++; acc->h1p += d.mix1; acc->h2p += d.mix2; acc->minBHp = min(acc->minBHp, bHp); }
        if (c >= L && c < H) acc->minBLlong = min(acc->minBLlong, c0 >= L ? 0u : bLp);   // in the band when the last batch starts
    }
    return word;
}

// first prefix batch (1-based) in which an observer with stored word `uo` has >= L reports: 0 = it already has, T32_NONE = not in the prefix
__device__ __forceinline__ uint32_t observer_L_batch(uint32_t uo, const SubjDesc* dobs, const SubjWalk* pwo, int L) {
    int c = __popc(uo);
    if (c >= L) return 0u;
    if (dobs == nullptr || dobs->pmask == 0) return T32_NONE;
    const int np = __popc(dobs->pmask);
    for (int q = 0; q < np; ++q) {
        if ((uo >> pwo->ring[q]) & 1u) continue;
        if (++c == L) return pwo->time[q];
    }
    return T32_NONE;
}

struct ApplyArgs {
    RowRef rows;                  // the double-buffered state rows (rows.cur: which of a slot's two rows is current)
    size_t Rpad;
    int K, H, L;
    int64_t R, rbegin;
    const uint32_t* rflags;
    DeliveryDev dl;
    const BatchCounts* bc;        // device counters of the batch in flight: the number of batch subjects, the first fresh slot
                                  // (slots >= S_before were assigned by this batch: known-zero state, never read) and the
                                  // overflow flag come from HERE — the host never learns them inside a batch
    const SubjDesc* desc;
    const SubjWalk* walk;
    const SubjWalk* pwalk;        // sequences of batches: prefix walks
    const int32_t* touch;         // [slot] serial of the last batch with a valid cell for the slot
    const int32_t* batch_index;   // [slot] -> index in the batch in flight (valid if touch[slot] == serial)
    int32_t serial;
    int seq;                      // a sequence of batches in one pass (SEQ kernels)
    const int32_t* slot_subject;
    const int32_t* sidx;          // sorted cell indices
    const uint8_t* s_ring;
    const uint8_t* s_status;
    Partials part;
    int n_tiles;
    WorkList wl;                  // invalidation work list
};

__device__ __forceinline__ void note_unresolved(const ApplyArgs& a, int tile, int32_t slot) { worklist_note(a.wl, tile, slot); }

// ---- uniform delivery: every active receiver gets every valid cell in array order -------------------------------------
// One thread owns 8 consecutive receivers: per subject one group load and one group store (RowRef: 64-bit lo plane + 16-bit hi
// plane at HB = 2, so a warp writes 256 + 64 bytes, all of them whole 32-byte sectors).  The common case is
// that all of a thread's ACTIVE receivers hold the same state for the subject (they saw the same history): the
// visit is computed once, merged into the new word with a SWAR mask, and accumulated in registers ("com").  Only
// when active neighbours disagree (partitions) do we fall back to a per-receiver visit whose accumulators live in
// the thread's own slice of the global partial arrays.
template <bool SEQ>
__device__ __forceinline__ void part_store(const Partials& p, size_t at, const Acc& a) {
    p.cnt[at] = make_uint4(a.nL, a.nH, a.tp | (a.flags << PF_SHIFT), a.nUn);
    if (SEQ) p.cntp[at] = make_uint4(a.nLp, a.nHp, a.tpc, 0u);
    p.minTH[at] = a.minTH == T32_NONE ? T64_NONE : (uint64_t)a.minTH;
    p.minTLun[at] = a.minTLun == T32_NONE ? T64_NONE : (uint64_t)a.minTLun;
    p.h1[at] = a.h1;
    p.h2[at] = a.h2;
    if (SEQ) { p.h1p[at] = a.h1p; p.h2p[at] = a.h2p; p.seq[at] = make_uint2(a.minBHp, a.minBLlong); }
}
template <bool SEQ>
__device__ __forceinline__ void part_merge(const Partials& p, size_t at, const Acc& a) {      // add `a` to what the slot holds
    uint4 c = p.cnt[at];
    c.x += a.nL; c.y += a.nH; c.z = (c.z + a.tp) | (a.flags << PF_SHIFT); c.w += a.nUn;
    p.cnt[at] = c;
    if (SEQ && (a.nLp | a.nHp | a.tpc)) { uint4 cp = p.cntp[at]; cp.x += a.nLp; cp.y += a.nHp; cp.z += a.tpc; p.cntp[at] = cp; }
    if (a.minTH != T32_NONE) { const uint64_t o = p.minTH[at]; if ((uint64_t)a.minTH < o) p.minTH[at] = a.minTH; }
    if (a.minTLun != T32_NONE) { const uint64_t o = p.minTLun[at]; if ((uint64_t)a.minTLun < o) p.minTLun[at] = a.minTLun; }
    if (a.nH) { p.h1[at] += a.h1; p.h2[at] += a.h2; }
    if (SEQ) {
        if (a.nHp) { p.h1p[at] += a.h1p; p.h2p[at] += a.h2p; }
        uint2 q = p.seq[at];
        q.x = min(q.x, a.minBHp); q.y = min(q.y, a.minBLlong);
        p.seq[at] = q;
    }
}

// Subjects whose slot was assigned by this very batch ("fresh") have known-zero state for EVERY receiver: nothing is
// read, the new word is the batch's ring mask under the thread's activity mask, and their contribution to the
// per-receiver accumulators is the same for every active receiver — it is reduced once per stage by warp 0 and added
// at the end.  Only carried subjects (reports from earlier batches) take the load / compare / visit path.
struct StageAcc {                     // one subject or one stage: the counts fit 16-bit halves (at most STAGE each)
    uint32_t nLH, tpUn, fl, minTH, minTLun;
    uint64_t h1, h2;
    uint32_t nLHp, tpc, minBHp, minBLlong;
    uint64_t h1p, h2p;
};

template <bool SEQ>
__device__ __forceinline__ StageAcc stage_pack(const Acc& f) {
    StageAcc s;
    s.nLH = f.nL | (f.nH << 16); s.tpUn = f.tp | (f.nUn << 16); s.fl = f.flags; s.minTH = f.minTH; s.minTLun = f.minTLun;
    s.h1 = f.h1; s.h2 = f.h2;
    s.nLHp = SEQ ? f.nLp | (f.nHp << 16) : 0u; s.tpc = SEQ ? f.tpc : 0u; s.minBHp = SEQ ? f.minBHp : T32_NONE;
    s.minBLlong = SEQ ? f.minBLlong : T32_NONE; s.h1p = SEQ ? f.h1p : 0ull; s.h2p = SEQ ? f.h2p : 0ull;
    return s;
}
// reduction of one record per lane over the warp (the result is valid in lane 0)
template <bool SEQ>
__device__ __forceinline__ StageAcc stage_reduce(StageAcc s) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s.nLH += __shfl_down_sync(0xffffffffu, s.nLH, o);
        s.tpUn += __shfl_down_sync(0xffffffffu, s.tpUn, o);
        s.fl |= __shfl_down_sync(0xffffffffu, s.fl, o);
        s.minTH = min(s.minTH, __shfl_down_sync(0xffffffffu, s.minTH, o));
        s.minTLun = min(s.minTLun, __shfl_down_sync(0xffffffffu, s.minTLun, o));
        s.h1 += __shfl_down_sync(0xffffffffu, s.h1, o);
        s.h2 += __shfl_down_sync(0xffffffffu, s.h2, o);
        if (SEQ) {
            s.nLHp += __shfl_down_sync(0xffffffffu, s.nLHp, o);
            s.tpc += __shfl_down_sync(0xffffffffu, s.tpc, o);
            s.minBHp = min(s.minBHp, __shfl_down_sync(0xffffffffu, s.minBHp, o));
            s.minBLlong = min(s.minBLlong, __shfl_down_sync(0xffffffffu, s.minBLlong, o));
            s.h1p += __shfl_down_sync(0xffffffffu, s.h1p, o);
            s.h2p += __shfl_down_sync(0xffffffffu, s.h2p, o);
        }
    }
    return s;
}
// c += the packed contribution of a whole stage (the chunk's sum needs the full 32-bit counts)
template <bool SEQ>
__device__ __forceinline__ void chunk_add(ChunkAcc& c, const StageAcc& m) {
    c.nL += m.nLH & 0xFFFFu; c.nH += m.nLH >> 16; c.tp += m.tpUn & 0xFFFFu; c.nUn += m.tpUn >> 16; c.fl |= m.fl;
    c.minTH = min(c.minTH, m.minTH); c.minTLun = min(c.minTLun, m.minTLun); c.h1 += m.h1; c.h2 += m.h2;
    if (SEQ) {
        c.nLp += m.nLHp & 0xFFFFu; c.nHp += m.nLHp >> 16; c.tpc += m.tpc; c.minBHp = min(c.minBHp, m.minBHp);
        c.minBLlong = min(c.minBLlong, m.minBLlong); c.h1p += m.h1p; c.h2p += m.h2p;
    }
}
__device__ __forceinline__ ChunkAcc chunk_zero() {
    ChunkAcc c;
    c.nL = 0; c.nH = 0; c.tp = 0; c.nUn = 0; c.fl = 0; c.minTH = T32_NONE; c.minTLun = T32_NONE; c.pad_ = 0; c.h1 = 0; c.h2 = 0;
    c.nLp = 0; c.nHp = 0; c.tpc = 0; c.minBHp = T32_NONE; c.minBLlong = T32_NONE; c.pad2_ = 0; c.h1p = 0; c.h2p = 0;
    return c;
}
// a += the packed contribution of one subject (or of a whole stage)
template <bool SEQ>
__device__ __forceinline__ void acc_add(Acc& a, const StageAcc& m) {
    a.nL += m.nLH & 0xFFFFu; a.nH += m.nLH >> 16; a.tp += m.tpUn & 0xFFFFu; a.nUn += m.tpUn >> 16; a.flags |= m.fl;
    a.minTH = min(a.minTH, m.minTH); a.minTLun = min(a.minTLun, m.minTLun); a.h1 += m.h1; a.h2 += m.h2;
    if (SEQ) {
        a.nLp += m.nLHp & 0xFFFFu; a.nHp += m.nLHp >> 16; a.tpc += m.tpc; a.minBHp = min(a.minBHp, m.minBHp);
        a.minBLlong = min(a.minBLlong, m.minBLlong); a.h1p += m.h1p; a.h2p += m.h2p;
    }
}

// One (subject, receiver) visit: [the prefix of a sequence,] then the (last) batch.  *word_out = the state when the last batch starts.
template <bool PERM, bool SEQ>
__device__ __forceinline__ bool visit_acc(Acc& acc, uint32_t ur, const SubjDesc& d, const SubjWalk* w, const SubjWalk* pw, uint32_t RM, int L, int H,
                                          const uint32_t* u = nullptr, uint32_t umask = 0, uint32_t last = 0, uint32_t* word_out = nullptr) {
    if (SEQ) ur = prefix_core(&acc, ur, d, *pw, u, umask, L, H, last);
    if (word_out) *word_out = ur;
    const Visit v = PERM ? visit_counts(ur & RM, d, RM, L, H) : visit_uniform(ur & RM, d, *w, L, H);
    return accumulate(acc, v, d, L, H);
}

// ---- dictionary observers of a subject ("edges"): when do they make the invalidation pass report a ring? ---------------------------
// RF_PRE_DOWN: finalize1 keeps the receiver's seenLinkDownEvents of BEFORE the call there (the passes after it recompute visits)
constexpr uint32_t RF_PRE_DOWN = 128u;
__device__ __forceinline__ uint32_t receiver_down_batch(const ApplyArgs& a, uint32_t rflag, bool after_finalize1) {
    if (rflag & (after_finalize1 ? RF_PRE_DOWN : RF_SEEN_DOWN)) return 0u;
    const int32_t sd = a.bc->seq_down;
    return sd == INT_MAX ? T32_NONE : (uint32_t)sd;
}
// pre-call row of a slot: before the flip it is the current one; after the flip the other one — for the slots the call touched
__device__ __forceinline__ const uint8_t* precall_row(const ApplyArgs& a, int32_t slot, bool post_flip) {
    const int flipped = post_flip && a.touch[slot] == a.serial ? 1 : 0;
    return a.rows.lo(slot, a.rows.cur[slot] ^ flipped);
}
// generic (one receiver, scalar loads): u[k] for every ring of `slot` whose observer is a subject itself; returns the ring mask
__device__ __noinline__ uint32_t edge_times(const ApplyArgs& a, int32_t slot, int64_t r, bool post_flip, uint32_t bDown, uint32_t* u) {
    if (!a.wl.has_so[slot]) return 0u;
    const uint32_t RM = (1u << a.K) - 1u;
    const int32_t S_before = a.bc->S_before;
    uint32_t umask = 0;
    for (int k = 0; k < a.K; ++k) {
        const int32_t so = a.wl.so_tab[(size_t)slot * SO_STRIDE + k];
        if (so < 0) continue;
        const bool ot = a.touch[so] == a.serial;
        const int bo = ot ? a.batch_index[so] : 0;
        const uint32_t uo = so >= S_before ? 0u : (a.rows.get(precall_row(a, so, post_flip), r) & RM);
        const uint32_t bLo = observer_L_batch(uo, ot ? &a.desc[bo] : nullptr, ot ? &a.pwalk[bo] : nullptr, a.L);
        u[k] = (bLo == T32_NONE || bDown == T32_NONE) ? T32_NONE : max(bLo, bDown);
        umask |= 1u << k;
    }
    return umask;
}
// state of (batch subject d, receiver r) when the last batch of the call starts, from its PRE-call word (passes that recompute visits)
__device__ __forceinline__ uint32_t seq_state(const ApplyArgs& a, const SubjDesc& d, int b_index, int64_t r, uint32_t old, bool post_flip,
                                              bool after_finalize1) {
    if (!a.seq) return old;
    uint32_t u[MAXK];
    const uint32_t umask = edge_times(a, d.slot, r, post_flip, receiver_down_batch(a, a.rflags[r], after_finalize1), u);
    if (umask == 0 && d.pmask == 0) return old;
    return prefix_core(nullptr, old, d, a.pwalk[b_index], u, umask, a.L, a.H, (uint32_t)a.bc->seq_last);
}

template <bool PERM, bool SEQ, int HB>
__global__ void __launch_bounds__(UNI_THREADS, UNI_MINBLOCKS) k_apply_uniform(const ApplyArgs a) {
    __shared__ SubjDesc sd[STAGE];
    __shared__ SubjWalk sw[PERM ? 1 : STAGE];
    __shared__ SubjWalk spw[SEQ ? STAGE : 1];
    __shared__ const uint8_t* s_src[STAGE];   // lo planes of the current / the other row
    __shared__ uint8_t* s_dst[STAGE];
    __shared__ uint32_t s_nw[STAGE];          // rings reported by the call
    __shared__ uint2 s_nrep[STAGE];           // ... replicated over the lanes (group8_rep)
    __shared__ int s_unres[STAGE];
    __shared__ ChunkAcc s_facc;               // fresh-subject accumulators of this block's chunk (same for every receiver)
    __shared__ int s_heavy;                   // staged subjects that are NOT plain fresh ones (carried, or with dictionary observers)
    // SEQ: the dictionary observers ("edges") of the staged subjects — their pre-call rows (nullptr: fresh, state 0) and batch index
    __shared__ uint8_t s_ne[SEQ ? STAGE : 1];
    __shared__ uint8_t s_ek[SEQ ? STAGE : 1][MAXK];
    __shared__ const uint8_t* s_erow[SEQ ? STAGE : 1][MAXK];
    __shared__ int32_t s_eob[SEQ ? STAGE : 1][MAXK];
    // Memo of the carried subjects: receivers of a tile have almost always seen the same history, so warp 0 computes
    // the visit ONCE per (block, subject) for the state the tile's first active receiver holds; a thread whose active receivers
    // all hold exactly that state only merges the precomputed new word, and takes the stage's summed contribution at the end of the
    // stage.  (The visit itself — the walk over the first-occurrence rings — was what kept the read-modify-write path issue-bound.)
    __shared__ uint32_t s_mst[STAGE];         // the sample state (0xFFFFFFFF: no memo for this subject)
    __shared__ uint2 s_mrep[STAGE];           // the new word for that state, replicated over the lanes
    __shared__ uint8_t s_mun[STAGE];          // the subject stays in the unstable band for that state
    __shared__ StageAcc s_macc[STAGE];        // what one such (subject, receiver) visit contributes
    __shared__ StageAcc s_msum;               // ... summed over the stage's memo subjects
    __shared__ uint32_t s_mall;               // which staged subjects have a memo
    __shared__ int s_wfirst[UNI_THREADS / 32];

    constexpr bool MEMO = !SEQ;               // (the sequence kernels keep the plain path: their visit depends on the observers' rows too)
    if (a.bc->overflow) return;               // the batch was rolled back by k_prepare
    // the number of batch subjects / the first fresh slot are only known on the device
    const int Sb = a.bc->n_batch_subj, S_before = a.bc->S_before;
    const int per_chunk = max(1, (Sb + (int)gridDim.y - 1) / (int)gridDim.y);
    const int tile = blockIdx.x, chunk = blockIdx.y, t = threadIdx.x;
    const int s0 = min(Sb, chunk * per_chunk), s1 = min(Sb, s0 + per_chunk);
    const int64_t r0 = (int64_t)tile * TILE_R + (int64_t)t * 8;
    const size_t pbase = (size_t)chunk * a.Rpad + (size_t)r0;
    const uint32_t RM = (1u << a.K) - 1u;
    const int L = a.L, H = a.H;
    const uint32_t seq_last = SEQ ? (uint32_t)a.bc->seq_last : 0u;

    uint32_t act = 0, seen = 0;               // seen: receivers whose seenLinkDownEvents is already set (SEQ)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int64_t r = r0 + j;
        if (r < a.R) {
            const uint32_t rf = a.rflags[r];
            const bool on = !(rf & RF_ANNOUNCED) && !((a.dl.flags & RAPID_DELIVERY_BLOCKED) && a.dl.blocked[r]);
            act |= (on ? 1u : 0u) << j;
            if (SEQ && (rf & RF_SEEN_DOWN)) seen |= 1u << j;
        }
    }
    const Group8<HB> am = group8_mask<HB>(act);     // SWAR masks: all-ones lanes of the active receivers
    const RowRef& rows = a.rows;
    if (t == 0) s_facc = chunk_zero();
    if (MEMO) {                                     // the tile's first active receiver
        const int mine = act ? t * 8 + __ffs(act) - 1 : INT_MAX;
        const int wmin = __reduce_min_sync(0xffffffffu, mine);
        if ((t & 31) == 0) s_wfirst[t >> 5] = wmin;
    }
    const int block_active = __syncthreads_or(act != 0);
    int sample_r = 0;
    if (MEMO && t < 32) {
        int f = INT_MAX;
#pragma unroll
        for (int q = 0; q < UNI_THREADS / 32; ++q) f = min(f, s_wfirst[q]);
        sample_r = f == INT_MAX ? 0 : f;
    }
    const size_t sample_at = (size_t)tile * TILE_R + (size_t)sample_r;
    Acc com;                                              // carried subjects: shared by all ACTIVE receivers of this thread
    bool had_exc = false;                                 // the thread's global partial slots hold per-receiver extras
    bool carried = false;                                 // this thread visited a carried subject (com is not just zeros)

    for (int base = s0; base < s1; base += STAGE) {
        const int n = min(STAGE, s1 - base);
        __syncthreads();
        if (t < 32) {                                     // warp 0 stages the descriptors (STAGE == 32)
            Acc f;                                        // what this lane's FRESH subject contributes to every active receiver
            Acc m;                                        // memo: what this lane's CARRIED subject contributes for the sample state
            bool heavy = false, memo = false;
            if (t < n) {
                const SubjDesc d = a.desc[base + t];
                sd[t] = d;
                const uint8_t c = rows.cur[d.slot];
                const bool fresh = d.slot >= S_before;
                s_src[t] = fresh ? nullptr : rows.lo(d.slot, c);
                s_dst[t] = rows.lo(d.slot, c ^ 1);
                s_nw[t] = (uint32_t)(d.bmask | d.pmask);
                s_nrep[t] = group8_rep<HB>(d.bmask | d.pmask);
                int un = 0;
                const bool edges = SEQ && a.wl.has_so[d.slot];   // implicit reports inside the prefix: per-receiver state matters
                if (SEQ) {
                    int ne = 0;
                    if (edges) {
                        for (int k = 0; k < a.K; ++k) {
                            const int32_t so = a.wl.so_tab[(size_t)d.slot * SO_STRIDE + k];
                            if (so < 0) continue;
                            s_ek[t][ne] = (uint8_t)k;
                            s_erow[t][ne] = so >= S_before ? nullptr : rows.cur_lo(so);
                            s_eob[t][ne] = a.touch[so] == a.serial ? a.batch_index[so] : -1;
                            ++ne;
                        }
                    }
                    s_ne[t] = (uint8_t)ne;
                }
                if (fresh && !edges) {
                    // state 0 for everyone: the descriptor-level answers (prefix_core / visit_uniform take their shortcuts)
                    un = (visit_acc<PERM, SEQ>(f, 0u, d, &sw[0], &spw[0], RM, L, H) && block_active) ? 1 : 0;   // (walks not read)
                    if (PERM) { f.minTH = T32_NONE; f.minTLun = T32_NONE; }
                } else {
                    if (!PERM) sw[t] = a.walk[base + t];
                    if (SEQ) spw[t] = a.pwalk[base + t];
                    if (fresh) s_src[t] = nullptr;
                    if (MEMO && !fresh && !edges && block_active) {
                        const uint32_t sst = rows.get(s_src[t], (int64_t)sample_at);
                        uint32_t at_last = sst;
                        const bool mun = visit_acc<PERM, SEQ>(m, sst & RM, d, &sw[PERM ? 0 : t], &spw[SEQ ? t : 0], RM, L, H, nullptr, 0u, seq_last, &at_last);
                        s_mst[t] = sst;
                        s_mrep[t] = group8_rep<HB>((SEQ ? at_last : sst) | s_nw[t]);
                        s_mun[t] = mun ? 1 : 0;
                        memo = true;
                    }
                }
                if (MEMO) { if (!memo) s_mst[t] = 0xFFFFFFFFu; else s_macc[t] = stage_pack<SEQ>(m); }
                // only subjects with an observer in the dictionary can receive implicit reports: the others never go on
                // the invalidation work list (has_so is refreshed by k_prepare whenever a subject gets a slot)
                s_unres[t] = (un && a.wl.has_so[d.slot]) ? 1 : 0;
                if (!fresh || edges) s_unres[t] = a.wl.has_so[d.slot] ? 0 : -1;       // -1: never list it
                heavy = !fresh || edges;
            }
            {
                const unsigned hm = __ballot_sync(0xffffffffu, heavy);
                if (t == 0) s_heavy = __popc(hm);
            }
            // warp reduction of the fresh subjects' contribution
            const StageAcc fr = stage_reduce<SEQ>(stage_pack<SEQ>(f));
            if (t == 0) chunk_add<SEQ>(s_facc, fr);
            if (MEMO) {
                const unsigned mm = __ballot_sync(0xffffffffu, memo);
                if (mm) {                                 // (warp-uniform)
                    const StageAcc mr = stage_reduce<SEQ>(stage_pack<SEQ>(m));
                    if (t == 0) s_msum = mr;
                }
                if (t == 0) s_mall = mm;
            }
        }
        __syncthreads();
        uint32_t hit = 0;                                  // staged subjects for which this thread took the memo
        // The read-modify-write path has ONE group load (both planes) in flight per thread (the loop body branches on the loaded
        // words), far below what the HBM latency-bandwidth product needs.  The rows of the next PF_DIST staged subjects are
        // therefore pulled into L2 ahead of their loads.
        const bool pf_on = !SEQ && s_heavy != 0;          // (the sequence kernels keep their measured code: no memo, no prefetch)
        if (pf_on) {
#pragma unroll
            for (int j = 0; j < PF_DIST; ++j)
                if (j < n && s_src[j]) {
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(s_src[j] + r0));
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(group8_hi<HB>(rows, s_src[j], r0)));
                }
        }
#pragma unroll 4
        for (int i = 0; i < n; ++i) {
            const uint8_t* src = s_src[i];
            uint8_t* dst = s_dst[i];
            const int ne = SEQ ? (int)s_ne[i] : 0;
            if (pf_on && i + PF_DIST < n) {
                const uint8_t* nx = s_src[i + PF_DIST];
                if (nx) {
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(nx + r0));
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(group8_hi<HB>(rows, nx, r0)));
                }
            }
            if (src == nullptr && ne == 0) {               // fresh subject: write-only, full width (zeros for inactive receivers)
                group8_store<HB>(rows, dst, r0, group8_fill<HB>(s_nrep[i], am));
                continue;
            }
            Group8<HB> w;
            if (src) w = group8_load<HB>(rows, src, r0);
            else { w.lo = 0; w.hi = 0; }
            bool unres = false;
            if (act) {
                const SubjDesc& d = sd[i];
                uint32_t st;
                bool same = group8_same<HB>(w, am, &st);     // all active receivers hold the same word
                carried = true;
                const bool mhit = MEMO && same && st == s_mst[i];   // (subjects with edges have no memo)
                // SEQ, subject with dictionary observers: their state (and seenLinkDownEvents) must be the same across the thread's
                // active receivers too, or every receiver is visited on its own
                uint32_t u[MAXK];
                uint32_t umask = 0;
                if (SEQ && ne && !mhit) {
                    const uint32_t sact = seen & act;
                    same = same && (sact == 0 || sact == act);
                    const uint32_t bDown = sact ? 0u : (a.bc->seq_down == INT_MAX ? T32_NONE : (uint32_t)a.bc->seq_down);
                    for (int e = 0; e < ne && same; ++e) {
                        uint32_t so_st = 0;
                        if (s_erow[i][e]) same = group8_same<HB>(group8_load<HB>(rows, s_erow[i][e], r0), am, &so_st);
                        const int ob = s_eob[i][e], k = s_ek[i][e];
                        const uint32_t bLo = observer_L_batch(so_st & RM, ob >= 0 ? &a.desc[ob] : nullptr, ob >= 0 ? &a.pwalk[ob] : nullptr, L);
                        u[k] = (bLo == T32_NONE || bDown == T32_NONE) ? T32_NONE : max(bLo, bDown);
                        umask |= 1u << k;
                    }
                }
                if (mhit) {                                // the tile's common state: everything is precomputed
                    hit |= 1u << i;
                    unres = s_mun[i] != 0;
                    group8_merge<HB>(w, s_mrep[i], am);
                } else if (same) {
                    uint32_t at_last = st;
                    unres = visit_acc<PERM, SEQ>(com, st & RM, d, &sw[PERM ? 0 : i], &spw[SEQ ? i : 0], RM, L, H, u, umask, seq_last, &at_last);
                    group8_merge<HB>(w, group8_rep<HB>((SEQ ? at_last : st) | s_nw[i]), am);
                } else {
                    if (!had_exc) {
                        had_exc = true;
                        const Acc zero;
#pragma unroll
                        for (int j = 0; j < 8; ++j) part_store<SEQ>(a.part, pbase + j, zero);
                    }
                    const uint32_t nwb = s_nw[i];
                    // (the sequence kernels keep this rare per-receiver path rolled: unrolled, it spills their hot loop)
#pragma unroll (SEQ ? 1 : 8)
                    for (int j = 0; j < 8; ++j) {
                        if (!((act >> j) & 1u)) continue;
                        const uint32_t sj = group8_word<HB>(w, j);
                        Acc ex;
                        uint32_t at_last = sj;
                        if (SEQ && ne) umask = edge_times(a, d.slot, r0 + j, false, receiver_down_batch(a, ((seen >> j) & 1u) ? RF_SEEN_DOWN : 0u, false), u);
                        unres |= visit_acc<PERM, SEQ>(ex, sj & RM, d, &sw[PERM ? 0 : i], &spw[SEQ ? i : 0], RM, L, H, u, umask, seq_last, &at_last);
                        part_merge<SEQ>(a.part, pbase + j, ex);
                        group8_or_word<HB>(w, j, (SEQ ? (at_last & RM) : 0u) | nwb);
                    }
                }
            }
            group8_store<HB>(rows, dst, r0, w);            // the non-current row becomes the new state
            if (__any_sync(0xffffffffu, unres) && (t & 31) == 0 && s_unres[i] == 0) s_unres[i] = 1;
        }
        if (MEMO && hit) {                           // the memo subjects this thread met: usually all of the stage's
            if (hit == s_mall) acc_add<SEQ>(com, s_msum);
            else for (uint32_t mh = hit; mh; mh &= mh - 1) acc_add<SEQ>(com, s_macc[__ffs(mh) - 1]);
        }
        __syncthreads();
        if (t < n && s_unres[t] > 0) note_unresolved(a, tile, sd[t].slot);
    }
    // Fresh subjects contribute the same to every active receiver: that goes to ONE record per chunk.  Per-receiver
    // partials are only written by blocks in which some thread met a carried subject; finalize1 adds the two.
    const int need = __syncthreads_or((carried || had_exc) ? 1 : 0);
    if (t == 0) {
        a.part.flag[(size_t)chunk * a.part.n_tiles + tile] = need;
        if (tile == 0) a.part.chunk[chunk] = s_facc;
    }
    if (!need) return;
    const Acc zero;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const size_t at = pbase + j;
        const bool on = (act >> j) & 1u;
        if (!had_exc) part_store<SEQ>(a.part, at, on ? com : zero);
        else if (on) part_merge<SEQ>(a.part, at, com);
    }
}

// ---- generic delivery (per-receiver subset and/or per-receiver order): one receiver per thread -------------------
struct GVisit {
    int c0, c1;
    bool crossL, crossH, seen_down;
    uint64_t tL, tH;
    uint32_t have;        // rings delivered to this receiver in this batch
};

// moments of a subject's cells as seen by one receiver; `rs` is the receiver's permutation seed
__device__ __forceinline__ GVisit visit_generic(uint32_t ur, const SubjDesc& d, const int32_t* __restrict__ sidx,
                                                const uint8_t* __restrict__ s_ring, const uint8_t* __restrict__ s_status,
                                                const DeliveryDev& dl, int64_t r, uint64_t rs, int L, int H) {
    GVisit v;
    v.have = 0; v.seen_down = false; v.tL = 0; v.tH = 0;
    const bool has_bitmap = dl.flags & RAPID_DELIVERY_BITMAP, permuted = dl.flags & RAPID_DELIVERY_PERMUTED;
    if (d.seg_len <= SMALL_SEG) {
        // Few cells (the common case: ~1-3 reports of a subject per batch): work on the cells themselves instead of a
        // per-ring table — first occurrence of each not-yet-reported ring, then its rank by moment, all in registers.
        uint64_t tm[SMALL_SEG];
        int rk[SMALL_SEG];
        bool ok[SMALL_SEG];
#pragma unroll
        for (int j = 0; j < SMALL_SEG; ++j) {
            ok[j] = false; tm[j] = 0; rk[j] = 0;
            if (j < (int)d.seg_len) {
                const int32_t ci = sidx[d.seg_begin + j];
                if (!has_bitmap || ((dl.bitmap[(size_t)ci * dl.words + (r >> 5)] >> (r & 31)) & 1u)) {
                    ok[j] = true;
                    rk[j] = s_ring[d.seg_begin + j];
                    tm[j] = permuted ? splitmix64(rs ^ (uint64_t)(ci - dl.cell_base)) : (uint64_t)ci + 1ull;
                    if (s_status[d.seg_begin + j] == RAPID_EDGE_DOWN) v.seen_down = true;
                    v.have |= 1u << rk[j];
                }
            }
        }
        const uint32_t fresh = v.have & ~ur;
        v.c0 = __popc(ur);
        v.c1 = v.c0 + __popc(fresh);
        v.crossL = v.c0 < L && v.c1 >= L;
        v.crossH = v.c0 < H && v.c1 >= H;
        if (v.crossL || v.crossH) {
            const int wantL = L - v.c0 - 1, wantH = H - v.c0 - 1;
            bool first[SMALL_SEG];
#pragma unroll
            for (int j = 0; j < SMALL_SEG; ++j) {             // first report of a ring this receiver had not counted yet
                first[j] = ok[j] && !((ur >> rk[j]) & 1u);
#pragma unroll
                for (int i = 0; i < SMALL_SEG; ++i)
                    if (i != j && ok[i] && rk[i] == rk[j] && tm[i] < tm[j]) first[j] = false;
            }
#pragma unroll
            for (int j = 0; j < SMALL_SEG; ++j) {
                if (!first[j]) continue;
                int rank = 0;
#pragma unroll
                for (int i = 0; i < SMALL_SEG; ++i) rank += (first[i] && tm[i] < tm[j]) ? 1 : 0;
                if (rank == wantL) v.tL = tm[j];
                if (rank == wantH) v.tH = tm[j];
            }
        }
        return v;
    }
    uint64_t tmin[MAXK];
#pragma unroll
    for (int k = 0; k < MAXK; ++k) tmin[k] = 0;
    const uint32_t e = d.seg_begin + d.seg_len;
    for (uint32_t j = d.seg_begin; j < e; ++j) {
        const int32_t ci = sidx[j];
        if (has_bitmap && !((dl.bitmap[(size_t)ci * dl.words + (r >> 5)] >> (r & 31)) & 1u)) continue;
        if (s_status[j] == RAPID_EDGE_DOWN) v.seen_down = true;
        const int k = s_ring[j];
        const uint64_t tm = permuted ? splitmix64(rs ^ (uint64_t)(ci - dl.cell_base)) : (uint64_t)ci + 1ull;
        const bool had = (v.have >> k) & 1u;
#pragma unroll
        for (int kk = 0; kk < MAXK; ++kk)
            if (kk == k && (!had || tm < tmin[kk])) tmin[kk] = tm;
        v.have |= 1u << k;
    }
    const uint32_t fresh = v.have & ~ur;
    v.c0 = __popc(ur);
    v.c1 = v.c0 + __popc(fresh);
    v.crossL = v.c0 < L && v.c1 >= L;
    v.crossH = v.c0 < H && v.c1 >= H;
    if (v.crossL || v.crossH) {
        const int wantL = L - v.c0 - 1, wantH = H - v.c0 - 1;       // rank (0-based) among the new rings' first moments
#pragma unroll
        for (int k = 0; k < MAXK; ++k) {
            if (!((fresh >> k) & 1u)) continue;
            int rank = 0;
#pragma unroll
            for (int q = 0; q < MAXK; ++q) rank += (((fresh >> q) & 1u) && tmin[q] < tmin[k]) ? 1 : 0;
            if (rank == wantL) v.tL = tmin[k];
            if (rank == wantH) v.tH = tmin[k];
        }
    }
    return v;
}

__global__ void __launch_bounds__(GEN_THREADS, 4) k_apply_generic(const ApplyArgs a) {
    __shared__ SubjDesc sd[STAGE];
    __shared__ const uint8_t* s_src[STAGE];
    __shared__ uint8_t* s_dst[STAGE];
    __shared__ int s_unres[STAGE];
    if (a.bc->overflow) return;               // the batch was rolled back by k_prepare
    const int Sb = a.bc->n_batch_subj, S_before = a.bc->S_before;
    const int per_chunk = max(1, (Sb + (int)gridDim.y - 1) / (int)gridDim.y);
    const int t = threadIdx.x, chunk = blockIdx.y;
    const int64_t r = (int64_t)blockIdx.x * GEN_THREADS + t;
    const int tile = (int)(((int64_t)blockIdx.x * GEN_THREADS) / TILE_R);
    const int s0 = min(Sb, chunk * per_chunk), s1 = min(Sb, s0 + per_chunk);
    const uint32_t RM = (1u << a.K) - 1u;
    const int L = a.L, H = a.H;
    const bool in_range = r < a.R;
    const bool active = in_range && !(a.rflags[r] & RF_ANNOUNCED) && !((a.dl.flags & RAPID_DELIVERY_BLOCKED) && a.dl.blocked[r]);
    const uint64_t rs = splitmix64(a.dl.perm_seed + (uint64_t)(a.rbegin + r));
    uint32_t nL = 0, nH = 0, tp = 0, nUn = 0, fl = 0;
    uint64_t minTH = T64_NONE, minTLun = T64_NONE, h1 = 0, h2 = 0;
    bool haveTH = false, haveTL = false;
    for (int base = s0; base < s1; base += STAGE) {
        const int n = min(STAGE, s1 - base);
        __syncthreads();
        if (t < n) {
            const SubjDesc d = a.desc[base + t];
            sd[t] = d;
            const uint8_t c = a.rows.cur[d.slot];
            s_src[t] = d.slot >= S_before ? nullptr : a.rows.lo(d.slot, c);
            s_dst[t] = a.rows.lo(d.slot, c ^ 1);
            s_unres[t] = a.wl.has_so[d.slot] ? 0 : -1;          // -1: no observer in the dictionary, never on the work list
        }
        __syncthreads();
        // the visit is a dependent chain (state word -> cells -> moments): keep 8 state loads in flight per thread
        uint32_t pre[8];
        for (int i = 0; i < n; ++i) {
            if ((i & 7) == 0) {
#pragma unroll
                for (int u = 0; u < 8; ++u) pre[u] = (i + u < n && s_src[i + u]) ? a.rows.get(s_src[i + u], r) : 0u;
            }
            const SubjDesc& d = sd[i];
            bool unres = false;
            if (r < (int64_t)a.Rpad) {
                uint32_t st = pre[i & 7];
                if (active) {
                    const GVisit v = visit_generic(st & RM, d, a.sidx, a.s_ring, a.s_status, a.dl, r, rs, L, H);
                    if (v.seen_down) fl |= PF_SEEN;
                    if (v.c0 >= L && v.c0 < H) tp++;
                    if (v.crossL) nL++;
                    if (v.crossH) {
                        nH++;
                        if (!haveTH || v.tH < minTH) { minTH = v.tH; haveTH = true; }
                        h1 += d.mix1; h2 += d.mix2;
                    }
                    if (v.c1 >= L && v.c1 < H) {
                        unres = true;
                        if (v.crossL) { nUn++; if (!haveTL || v.tL < minTLun) { minTLun = v.tL; haveTL = true; } }
                        else fl |= PF_NEGINF;
                    }
                    st |= v.have;
                }
                // (r < Rpad holds for the whole grid: every lane of the warp takes part in the store)
                if (a.rows.hb == 2) row_store1_warp<2>(a.rows, s_dst[i], r, st);
                else row_store1_warp<8>(a.rows, s_dst[i], r, st);
            }
            if (__any_sync(0xffffffffu, unres) && (t & 31) == 0 && s_unres[i] == 0) s_unres[i] = 1;
        }
        __syncthreads();
        if (t < n && s_unres[t] > 0) note_unresolved(a, tile, sd[t].slot);   // a 256-receiver block lies inside one tile
    }
    if (t == 0) {
        if ((blockIdx.x * GEN_THREADS) % TILE_R == 0) a.part.flag[(size_t)chunk * a.part.n_tiles + tile] = 1;
        if (blockIdx.x == 0) a.part.chunk[chunk] = chunk_zero();
    }
    if (r < (int64_t)a.Rpad) {
        const size_t p = (size_t)chunk * a.Rpad + (size_t)r;
        a.part.cnt[p] = make_uint4(nL, nH, tp | (fl << PF_SHIFT), nUn);
        a.part.minTH[p] = minTH;
        a.part.minTLun[p] = minTLun;
        a.part.h1[p] = h1;
        a.part.h2[p] = h2;
    }
}

// ==================================================================================================================
// k_resolve: everything after the apply kernel, in ONE cooperative launch (grid-wide barriers instead of host round trips)
//
//   finalize1   combine the chunk partials of every receiver, classify (EMIT_ALL / nothing / needs moments / MIXED)
//   [moments]   PERMUTED delivery only, flagged receivers only: their own min t_H / min t_L from the PRE-batch rows
//   [mixed]     exact interval analysis to its fixpoint (see below), flagged receivers only
//   flip        the rows written by the apply kernel become current
//   inval       invalidateFailingEdges over the (tile, subject) work list
//   finalize2   emissions of the invalidation pass, announced flags
//   [marks]     emit marks for receivers that announced only the explicit part
//   tail        the last block snapshots the batch counters for the host and resets the per-batch fields
// ==================================================================================================================
struct ResolveArgs {
    ApplyArgs ap;
    MarkPlane emit;               // bit 15 of the logical words (see MarkPlane)
    MarkPlane trans;              // bit 14: raised by this batch's invalidation pass
    BatchCounts* bc;
    BatchCounts* snap;
    int n_chunks;                 // subject chunks of the apply launch (layout of the partials)
    int uniform;                  // moments are cell indices (no PERMUTED / BITMAP)
    int counts_only;              // the apply kernel left the moments out (k_apply_uniform<true>)
    int seq;                      // a sequence of batches applied in one pass (prefix folded into the state, see visit_prefix)
    uint8_t* seq_dev;             // [Rpad] scratch of k_seq_check
    uint8_t* cur_w;
    int32_t* n_pre;
    uint32_t* rflags;
    uint64_t* pend_h1;
    uint64_t* pend_h2;
    int32_t* pend_cnt;
    uint64_t* out_h1;
    uint64_t* out_h2;
    int32_t* out_len;
    uint8_t* out_ann;
    uint32_t* mx_fl;
    uint64_t* mx_a;
    uint64_t* mx_cand;
    uint64_t* mx_emax;
    uint64_t* mx_p1;
    uint64_t* mx_p2;
    int32_t* mx_pc;
    uint64_t* estar;
    unsigned long long* mx_e1;
    unsigned long long* mx_e2;
    int32_t* mx_ec;
    int32_t* mx_changed;          // [4]
    uint32_t* mx_dev;             // [Rpad / 32] scratch of the reference-receiver shortcut (all zero between batches)
    const int32_t* slot_of;
    const int32_t* obs;
    const int32_t* touch;
    const int32_t* batch_index;
    int32_t serial;
    int inv_split;                // blocks per 1024-receiver tile in k_inval_finalize2 (1: a block walks the whole work list)
    int32_t* inv_res;             // [Rpad] subjects raised to >= H by the pass, summed over the blocks of a tile
    unsigned long long* inv_h1;   // [Rpad] their fingerprint sums
    unsigned long long* inv_h2;
    int32_t* inv_ticket;          // [n_tiles] blocks of the tile that have handed their part over
};

__device__ __forceinline__ int32_t block_sum_i32(int32_t v, int32_t* s_red) {      // every thread gets the block total
    __syncthreads();
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    int32_t s = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += s_red[w];
    return s;
}

// ------------------------------------------------------------------------------------------------------------------
// finalize 1: combine the chunk partials of every receiver, classify, keep the scalars
// ------------------------------------------------------------------------------------------------------------------
// What the FRESH subjects of the batch contribute is the same for every active receiver (one ChunkAcc per chunk of the apply
// launch): reduced once per block (warp 0) instead of once per receiver.
__device__ __forceinline__ void reduce_fresh(const ResolveArgs& a, ChunkAcc* s_fresh, int* s_fhave) {
    const ApplyArgs& ap = a.ap;
    if (threadIdx.x < 32) {
        uint32_t nL = 0, nH = 0, tp = 0, nUn = 0, fl = 0, mTH = T32_NONE, mTL = T32_NONE;
        uint64_t h1 = 0, h2 = 0;
        uint32_t nLp = 0, nHp = 0, tpc = 0, mBH = T32_NONE, mBL = T32_NONE;
        uint64_t h1p = 0, h2p = 0;
        for (int c = threadIdx.x; c < a.n_chunks; c += 32) {
            const ChunkAcc k = ap.part.chunk[c];
            nL += k.nL; nH += k.nH; tp += k.tp; nUn += k.nUn; fl |= k.fl;
            if (k.nH) mTH = min(mTH, k.minTH);
            if (k.nUn) mTL = min(mTL, k.minTLun);
            h1 += k.h1; h2 += k.h2;
            if (a.seq) {
                nLp += k.nLp; nHp += k.nHp; tpc += k.tpc; mBH = min(mBH, k.minBHp); mBL = min(mBL, k.minBLlong);
                h1p += k.h1p; h2p += k.h2p;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            nL += __shfl_down_sync(0xffffffffu, nL, o); nH += __shfl_down_sync(0xffffffffu, nH, o);
            tp += __shfl_down_sync(0xffffffffu, tp, o);
            nUn += __shfl_down_sync(0xffffffffu, nUn, o); fl |= __shfl_down_sync(0xffffffffu, fl, o);
            mTH = min(mTH, __shfl_down_sync(0xffffffffu, mTH, o)); mTL = min(mTL, __shfl_down_sync(0xffffffffu, mTL, o));
            h1 += __shfl_down_sync(0xffffffffu, h1, o); h2 += __shfl_down_sync(0xffffffffu, h2, o);
            nLp += __shfl_down_sync(0xffffffffu, nLp, o); nHp += __shfl_down_sync(0xffffffffu, nHp, o);
            tpc += __shfl_down_sync(0xffffffffu, tpc, o);
            mBH = min(mBH, __shfl_down_sync(0xffffffffu, mBH, o)); mBL = min(mBL, __shfl_down_sync(0xffffffffu, mBL, o));
            h1p += __shfl_down_sync(0xffffffffu, h1p, o); h2p += __shfl_down_sync(0xffffffffu, h2p, o);
        }
        if (threadIdx.x == 0) {
            ChunkAcc f;
            f.nL = nL; f.nH = nH; f.tp = tp; f.nUn = nUn; f.fl = fl; f.minTH = mTH; f.minTLun = mTL; f.pad_ = 0; f.h1 = h1; f.h2 = h2;
            f.nLp = nLp; f.nHp = nHp; f.tpc = tpc; f.minBHp = mBH; f.minBLlong = mBL; f.pad2_ = 0; f.h1p = h1p; f.h2p = h2p;
            *s_fresh = f;
            *s_fhave = (nH ? 1 : 0) | (nUn ? 2 : 0);
        }
    }
    __syncthreads();
}

__device__ void phase_finalize1(const ResolveArgs& a, int32_t* s_red) {
    const ApplyArgs& ap = a.ap;
    const int any_down = a.bc->any_down;
    __shared__ ChunkAcc s_fresh;
    __shared__ int s_fhave;
    reduce_fresh(a, &s_fresh, &s_fhave);
    int32_t my_mixed = 0, my_times = 0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < ap.R; r += (int64_t)gridDim.x * blockDim.x) {
        a.mx_fl[r] = 0;
        uint32_t flags = a.rflags[r] & ~(RF_ANN_NOW | RF_K3 | RF_ACTIVE | RF_PRE_DOWN);
        if (flags & RF_SEEN_DOWN) flags |= RF_PRE_DOWN;                 // seenLinkDownEvents as it was before this call
        a.out_h1[r] = 0; a.out_h2[r] = 0; a.out_len[r] = 0;
        const bool active = !(flags & RF_ANNOUNCED) && !((ap.dl.flags & RAPID_DELIVERY_BLOCKED) && ap.dl.blocked[r]);
        if (!active) { a.rflags[r] = flags; a.out_ann[r] = (flags & RF_ANNOUNCED) ? 1 : 0; continue; }
        flags |= RF_ACTIVE;
        uint32_t nL = s_fresh.nL, nH = s_fresh.nH, tp = s_fresh.tp, nUn = s_fresh.nUn, fl = s_fresh.fl;
        uint64_t minTH = s_fresh.minTH, minTLun = s_fresh.minTLun, h1 = s_fresh.h1, h2 = s_fresh.h2;
        uint32_t nLp = s_fresh.nLp, nHp = s_fresh.nHp;                                      // sequences: what the prefix did
        uint64_t h1p = s_fresh.h1p, h2p = s_fresh.h2p;
        bool haveTH = s_fhave & 1, haveTL = (s_fhave & 2) != 0;
        const int tile = (int)(r / TILE_R);
        // per-receiver partials of the chunks that met a carried subject: four chunks' loads in flight at a time
        for (int c0 = 0; c0 < a.n_chunks; c0 += 4) {
            int on[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) on[q] = c0 + q < a.n_chunks ? ap.part.flag[(size_t)(c0 + q) * ap.part.n_tiles + tile] : 0;
            uint4 q4[4], p4[4];
            uint64_t th[4], tl[4], a1[4], a2[4], b1[4], b2[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (!on[q]) continue;
                const size_t p = (size_t)(c0 + q) * ap.Rpad + (size_t)r;
                q4[q] = ap.part.cnt[p]; a1[q] = ap.part.h1[p]; a2[q] = ap.part.h2[p];
                if (!a.counts_only) { th[q] = ap.part.minTH[p]; tl[q] = ap.part.minTLun[p]; }
                if (a.seq) { p4[q] = ap.part.cntp[p]; b1[q] = ap.part.h1p[p]; b2[q] = ap.part.h2p[p]; }
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (!on[q]) continue;
                const uint32_t cH = q4[q].y, cUn = q4[q].w;
                nL += q4[q].x; nH += cH; tp += q4[q].z & TP_MASK; nUn += cUn; fl |= q4[q].z >> PF_SHIFT;
                if (!a.counts_only) {
                    if (cH && (!haveTH || th[q] < minTH)) { minTH = th[q]; haveTH = true; }
                    if (cUn && (!haveTL || tl[q] < minTLun)) { minTLun = tl[q]; haveTL = true; }
                }
                h1 += a1[q]; h2 += a2[q];
                if (a.seq) { nLp += p4[q].x; nHp += p4[q].y; h1p += b1[q]; h2p += b2[q]; }
            }
        }
        // every valid cell reaches every active receiver unless there is a per-receiver bitmap
        if ((a.uniform || a.counts_only) ? any_down : (fl & PF_SEEN)) flags |= RF_SEEN_DOWN;
        // a sequence of batches: the prefix moved nLp subjects into the band and nHp on to `proposal` before the last batch started
        const int32_t npre_old = a.n_pre[r] + (int32_t)nLp - (int32_t)nHp;
        const int32_t npre_new = npre_old + (int32_t)nL - (int32_t)nH;
        const uint64_t p1_old = a.pend_h1[r] + h1p, p2_old = a.pend_h2[r] + h2p;
        const int32_t pc_old = a.pend_cnt[r] + (int32_t)nHp;
        uint64_t ph1 = p1_old + h1, ph2 = p2_old + h2;
        int32_t pc = pc_old + (int32_t)nH;
        const int32_t untouched_pre = npre_old - (int32_t)tp;
        if (nH > 0 && npre_new == 0) {
            // EMIT_ALL: the last H-crossing of the batch leaves updatesInProgress == 0, so every subject at >= H has
            // left in some proposal of this batch (MultiNodeCutDetector.java:110-121); the union is what is announced.
            a.out_h1[r] = ph1; a.out_h2[r] = ph2; a.out_len[r] = pc;
            ph1 = 0; ph2 = 0; pc = 0;
            flags |= RF_ANNOUNCED | RF_ANN_NOW | RF_RULE_GE_H;
        } else if (nH > 0 && untouched_pre <= 0 && !(fl & PF_NEGINF)) {
            // every unresolved subject entered the band inside this batch: whether an H-crossing came before the first of
            // them depends on the moments (haveTL holds: npre_new > 0)
            if (a.counts_only) {
                // PERMUTED: the moments are this receiver's own — computed on demand from the pre-batch rows
                ++my_times;
                a.mx_fl[r] = MX_TIME;
                a.mx_a[r] = T64_NONE; a.mx_cand[r] = T64_NONE; a.mx_emax[r] = 0;
                a.mx_p1[r] = p1_old; a.mx_p2[r] = p2_old; a.mx_pc[r] = pc_old;
            } else if (!(haveTL && minTLun < minTH)) {
                // MIXED: some proposals may have been emitted before the unresolved subjects entered the band
                ++my_mixed;
                atomicMin(&a.bc->mx_first, (int32_t)r);              // candidate reference receiver of the interval analysis
                a.mx_fl[r] = MX_ON;
                a.mx_a[r] = minTLun; a.mx_cand[r] = T64_NONE; a.mx_emax[r] = 0;
                a.mx_p1[r] = p1_old; a.mx_p2[r] = p2_old; a.mx_pc[r] = pc_old;
            }
        }
        if (npre_new > 0 && (flags & RF_SEEN_DOWN)) flags |= RF_K3;
        a.n_pre[r] = npre_new;
        a.pend_h1[r] = ph1; a.pend_h2[r] = ph2; a.pend_cnt[r] = pc;
        a.rflags[r] = flags;
    }
    const int32_t bm = block_sum_i32(my_mixed, s_red), bt = block_sum_i32(my_times, s_red);
    if (threadIdx.x == 0) {
        if (bm) atomicAdd(&a.bc->n_mixed, bm);
        if (bt) atomicAdd(&a.bc->n_times, bt);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// MIXED receivers: exact interval analysis as data-parallel passes over (batch subjects x receivers).
//
// For one receiver the batch's subjects give intervals [t_L, t_H) (t_L = "before the batch" if the subject started
// inside the band, t_H = never if it does not reach H).  A proposal is emitted at t_H(s) iff no other interval covers
// it.  Let a = start of the connected component of intervals that contains the never-closing ones: everything closing
// after `a` is covered, and e* = the latest closing moment before `a` is the last explicit emission; what left is
// {t_H <= e*} plus whatever was pending before the batch.  `a` is found as a fixpoint: a <- min{t_L : t_H > a},
// starting from the earliest never-closing start (finalize1).  One FIX pass recomputes every flagged receiver's
// intervals from the PRE-batch rows (nothing is stored per (subject, receiver)); uniform delivery typically makes
// every receiver MIXED in the same way, so the passes are shaped like the apply kernels, not like a rare fallback.
// The loop runs on the device: pass, grid barrier, update, grid barrier, until no receiver's component grew.
// ------------------------------------------------------------------------------------------------------------------
struct IVisit { int c0, c1; bool crossL, crossH; uint64_t tL, tH; };

__device__ __forceinline__ IVisit interval_visit(const ApplyArgs& a, int uniform, uint32_t ur, const SubjDesc& d, const SubjWalk* w,
                                                 int64_t r, uint64_t rs) {
    IVisit o;
    if (uniform) {
        const Visit v = visit_uniform(ur, d, *w, a.L, a.H);
        o.c0 = v.c0; o.c1 = v.c1; o.crossL = v.crossL; o.crossH = v.crossH; o.tL = v.tL; o.tH = v.tH;
    } else {
        const GVisit v = visit_generic(ur, d, a.sidx, a.s_ring, a.s_status, a.dl, r, rs, a.L, a.H);
        o.c0 = v.c0; o.c1 = v.c1; o.crossL = v.crossL; o.crossH = v.crossH; o.tL = v.tL; o.tH = v.tH;
    }
    return o;
}

struct PassSmem {
    SubjDesc sd[STAGE];
    SubjWalk sw[STAGE];
    const uint8_t* s_old[STAGE];
};

// MODE 0: FIX pass (next candidate for `a`, e* candidate)   1: SUM pass (fingerprint of {t_H <= e*})
// MODE 2: MOMENT pass (min t_H over H-crossers -> mx_cand, min t_L over subjects left in the band -> mx_a)
template <int MODE>
__device__ __noinline__ void mixed_pass(const ResolveArgs& m, PassSmem& sm, const int Sb, const int S_before, const int64_t only_r = -1) {
    const ApplyArgs& a = m.ap;
    const int t = threadIdx.x;
    const uint32_t RM = (1u << a.K) - 1u;
    const int L = a.L, H = a.H;
    const int rblocks = (int)(a.Rpad / GEN_THREADS);
    int mchunks = max(1, min((Sb + STAGE - 1) / STAGE, (2 * (int)gridDim.x + rblocks - 1) / rblocks));
    const int mchunk = max(1, (Sb + mchunks - 1) / mchunks);
    mchunks = (Sb + mchunk - 1) / mchunk;
    const int64_t items = (int64_t)rblocks * mchunks;
    for (int64_t wi = blockIdx.x; wi < items; wi += gridDim.x) {
        const int rb = (int)(wi % rblocks), chunk = (int)(wi / rblocks);
        const int64_t r = (int64_t)rb * GEN_THREADS + t;
        const uint32_t fl = r < a.R ? m.mx_fl[r] : 0u;
        const bool on = (only_r < 0 || r == only_r) &&
                        (MODE == 0 ? ((fl & MX_ON) && !(fl & MX_DONE)) : MODE == 1 ? ((fl & MX_DONE) && (fl & MX_HAS_E) && !(fl & MX_REF)) : ((fl & MX_TIME) != 0));
        if (!__syncthreads_or(on ? 1 : 0)) continue;
        const uint64_t ref = on ? (MODE == 0 ? m.mx_a[r] : MODE == 1 ? m.estar[r] : 0ull) : 0ull;
        const uint64_t rs = splitmix64(a.dl.perm_seed + (uint64_t)(a.rbegin + r));
        const int s0 = chunk * mchunk, s1 = min(Sb, s0 + mchunk);
        uint64_t cand = T64_NONE, emax = 0, h1 = 0, h2 = 0, mTH = T64_NONE, mTL = T64_NONE;
        bool neg = false, has_e = false;
        int cnt = 0;
        for (int base = s0; base < s1; base += STAGE) {
            const int n = min(STAGE, s1 - base);
            __syncthreads();
            if (t < n) {
                const SubjDesc d = a.desc[base + t];
                sm.sd[t] = d;
                const bool fresh = d.slot >= S_before;
                sm.s_old[t] = fresh ? nullptr : a.rows.cur_lo(d.slot);   // pre-batch row (not flipped yet)
                if (!fresh && m.uniform) sm.sw[t] = a.walk[base + t];
            }
            __syncthreads();
            if (!on) continue;
            for (int i = 0; i < n; ++i) {
                const SubjDesc& d = sm.sd[i];
                const uint32_t st = seq_state(a, d, base + i, r, (sm.s_old[i] ? a.rows.get(sm.s_old[i], r) : 0u) & RM, false, true);   // when the (last) batch starts
                const IVisit v = interval_visit(a, m.uniform, st & RM, d, &sm.sw[i], r, rs);
                if (MODE == 0) {
                    if (!v.crossH) continue;                                  // never closes, or never in the band
                    const bool starts_in = v.c0 >= L && v.c0 < H;
                    if (v.tH > ref) { if (starts_in) neg = true; else if (v.tL < cand) cand = v.tL; }
                    else if (!has_e || v.tH > emax) { emax = v.tH; has_e = true; }
                } else if (MODE == 1) {
                    if (v.crossH && v.tH <= ref) { h1 += d.mix1; h2 += d.mix2; ++cnt; }
                } else {
                    if (v.crossH && v.tH < mTH) mTH = v.tH;
                    if (v.crossL && v.c1 < H && v.tL < mTL) mTL = v.tL;
                }
            }
        }
        if (!on) continue;
        if (MODE == 0) {
            if (neg) atomicOr(&m.mx_fl[r], MX_NEG);
            if (cand != T64_NONE) atomicMin((unsigned long long*)&m.mx_cand[r], (unsigned long long)cand);
            if (has_e) { atomicMax((unsigned long long*)&m.mx_emax[r], (unsigned long long)emax); atomicOr(&m.mx_fl[r], MX_HAS_E); }
        } else if (MODE == 1) {
            if (cnt) { atomicAdd(&m.mx_e1[r], (unsigned long long)h1); atomicAdd(&m.mx_e2[r], (unsigned long long)h2); atomicAdd(&m.mx_ec[r], cnt); }
        } else {
            if (mTH != T64_NONE) atomicMin((unsigned long long*)&m.mx_cand[r], (unsigned long long)mTH);
            if (mTL != T64_NONE) atomicMin((unsigned long long*)&m.mx_a[r], (unsigned long long)mTL);
        }
    }
}

// after the MOMENT pass: an unresolved subject entered the band before the first H-crossing -> nothing was emitted; else MIXED
__device__ void phase_classify_moments(const ResolveArgs& a, int32_t* s_red) {
    int32_t my_mixed = 0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.ap.R; r += (int64_t)gridDim.x * blockDim.x) {
        if (!(a.mx_fl[r] & MX_TIME)) continue;
        const uint64_t tl = a.mx_a[r], th = a.mx_cand[r];
        if (tl < th) { a.mx_fl[r] = 0; continue; }
        a.mx_fl[r] = MX_ON; a.mx_cand[r] = T64_NONE; a.mx_emax[r] = 0;
        ++my_mixed;
    }
    const int32_t bm = block_sum_i32(my_mixed, s_red);
    if (threadIdx.x == 0 && bm) atomicAdd(&a.bc->n_mixed, bm);
}

__device__ void phase_mixed_update(const ResolveArgs& a, int32_t* changed, int32_t* s_red, const int64_t only_r = -1) {
    int32_t my = 0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.ap.R; r += (int64_t)gridDim.x * blockDim.x) {
        if (only_r >= 0 && r != only_r) continue;
        const uint32_t fl = a.mx_fl[r];
        if (!(fl & MX_ON) || (fl & MX_DONE)) continue;
        if (fl & MX_NEG) { a.mx_fl[r] = 0; continue; }           // covered since before the batch: nothing was emitted
        const uint64_t c = a.mx_cand[r];
        if (c < a.mx_a[r]) {                                      // the component grows leftwards: another pass
            a.mx_a[r] = c; a.mx_cand[r] = T64_NONE; a.mx_emax[r] = 0; a.mx_fl[r] = fl & ~MX_HAS_E;
            ++my;
        } else if (fl & MX_HAS_E) {
            a.estar[r] = a.mx_emax[r];
            a.mx_fl[r] = fl | MX_DONE;
        } else {
            a.mx_fl[r] = 0;                                       // no closing moment before the component: nothing emitted
        }
    }
    const int32_t b = block_sum_i32(my, s_red);
    if (threadIdx.x == 0 && b) atomicAdd(changed, b);
}

__device__ void phase_mixed_commit(const ResolveArgs& a) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.ap.R; r += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t fl = a.mx_fl[r];
        if (!((fl & MX_DONE) && (fl & MX_HAS_E))) continue;
        // what left explicitly = everything pending before the batch + the batch subjects that closed by e*
        const uint64_t o1 = a.mx_p1[r] + a.mx_e1[r], o2 = a.mx_p2[r] + a.mx_e2[r];
        const int32_t oc = a.mx_pc[r] + a.mx_ec[r];
        a.out_h1[r] = o1; a.out_h2[r] = o2; a.out_len[r] = oc;
        a.pend_h1[r] -= o1; a.pend_h2[r] -= o2; a.pend_cnt[r] -= oc;
        a.mx_e1[r] = 0; a.mx_e2[r] = 0; a.mx_ec[r] = 0;
        a.rflags[r] = (a.rflags[r] | RF_ANNOUNCED | RF_ANN_NOW | RF_MIXED_EMIT) & ~RF_RULE_GE_H;
    }
}

// Did subject slot `s` leave in an explicit proposal of the batch in flight, for an RF_MIXED_EMIT receiver?  Rows have been
// flipped: the pre-batch row is the non-current one.
__device__ __noinline__ bool emitted_in_batch(const ResolveArgs& e, int32_t s, int64_t r, uint32_t w_new, uint64_t rs) {
    const ApplyArgs& a = e.ap;
    const uint32_t RM = (1u << a.K) - 1u;
    // untouched by the batch: it left (with the first explicit proposal) iff it was pending, i.e. at >= H and NOT raised there by
    // this batch's invalidation pass (the transient plane, cleared by the unmark phase once the batch is done)
    if (e.touch[s] != e.serial) return __popc(w_new & RM) >= a.H && !e.trans.test(s, r);
    const int b = e.batch_index[s];
    const SubjDesc d = a.desc[b];
    const uint32_t old = seq_state(a, d, b, r, (s >= a.bc->S_before ? 0u : a.rows.get(a.rows.alt_lo(s), r)) & RM, true, true);
    if (__popc(old & RM) >= a.H) return true;                              // pending before the (last) batch
    SubjWalk wl;
    if (e.uniform) wl = a.walk[b];
    const IVisit v = interval_visit(a, e.uniform, old & RM, d, &wl, r, rs);
    return v.crossH && v.tH <= e.estar[r];
}

// ------------------------------------------------------------------------------------------------------------------
// invalidateFailingEdges (MultiNodeCutDetector.java:137-164) + the receiver's closing bookkeeping, per 256-receiver unit.
// The work list names the subjects that sit in the unstable band of some receiver AND have an observer that is itself a
// subject; a unit walks the list (skipping subjects not in the band anywhere in its 1024-receiver tile), ORs in the implicit
// reports from observers that are themselves in proposal U preProposal, and — since everything a receiver needs is now in
// the thread's registers — finishes the receiver right away: emissions of the pass, announced flags, outputs.
// ------------------------------------------------------------------------------------------------------------------
constexpr int INV_STAGE = 128;            // work-list subjects staged at a time: one thread each (GEN_THREADS >= INV_STAGE)
struct InvSmem {
    uint8_t* row[INV_STAGE];                        // lo planes of the current rows
    uint64_t mix1[INV_STAGE], mix2[INV_STAGE];
    uint8_t ne[INV_STAGE];                          // edges (observers that are subjects) of staged slot i: entries [i * MAXK, i * MAXK + ne[i])
    const uint8_t* e_row[INV_STAGE * MAXK];
    int32_t e_so[INV_STAGE * MAXK];
    uint8_t e_k[INV_STAGE * MAXK];
    uint8_t flag[INV_STAGE];
    uint8_t dense[INV_STAGE];                       // the staged slots that are in the band somewhere in this tile
    int32_t n_dense;
};

// A block owns one 1024-receiver tile at a time, a thread 4 consecutive receivers (64-bit row loads, 128-bit flag loads).
// MX == false: every receiver EXCEPT those that announced through the interval analysis in this batch (RF_MIXED_EMIT) — the
// common case, no out-of-line call in the loop.  MX == true (k_marks, only when some receiver is MIXED): exactly those receivers;
// for them an observer that already left in an explicit proposal of this batch is no longer in `proposal` (emitted_in_batch).
template <bool MX>
__device__ void phase_inval_finalize2(const ResolveArgs& e, int mixed, InvSmem& sm, int32_t* s_red) {
    static_assert(TILE_R == 4 * GEN_THREADS, "a thread owns 4 receivers of a tile");
    const ApplyArgs& a = e.ap;
    const uint32_t RM = (1u << a.K) - 1u;
    const int t = threadIdx.x;
    const int n_list = min(*(volatile int32_t*)a.wl.count, a.wl.cap);
    int32_t my_inval = 0;
    // Small clusters have few tiles and one block per tile would walk the whole list alone (C3: 10 blocks x ~125 dependent
    // iterations).  The pass is independent per subject — an observer's membership in proposal U preProposal does not
    // change while it runs (implicit reports only move subjects from the band to >= H) — so P blocks share a tile: each takes a
    // contiguous part of the list, adds what it raised to per-receiver accumulators, and the last one to finish closes the receivers.
    const int P = MX ? 1 : max(1, e.inv_split);
    __shared__ int s_fin;
    for (int tb = blockIdx.x; tb < a.n_tiles * P; tb += gridDim.x) {
        const int tile = P > 1 ? tb % a.n_tiles : tb;
        int lo = 0, hi = n_list;
        if (P > 1) {
            const int per = max(8, (n_list + P - 1) / P);
            lo = min(n_list, (tb / a.n_tiles) * per); hi = min(n_list, lo + per);
        }
        const int64_t rb = (int64_t)tile * TILE_R + (int64_t)t * 4;
        const uint4 rf4 = *reinterpret_cast<const uint4*>(e.rflags + rb);          // rows and flags are padded to whole tiles
        uint32_t flags[4] = {rf4.x, rf4.y, rf4.z, rf4.w};
        bool k3[4];
        bool any_k3 = false;
        bool mine[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            mine[j] = rb + j < a.R && (((flags[j] & RF_MIXED_EMIT) != 0 && mixed) == MX);
            k3[j] = mine[j] && (flags[j] & RF_ACTIVE) && (flags[j] & RF_K3);
            any_k3 |= k3[j];
        }
        int32_t res[4] = {0, 0, 0, 0};
        uint64_t kh1[4] = {0, 0, 0, 0}, kh2[4] = {0, 0, 0, 0};
        if (n_list > 0 && __syncthreads_or(any_k3 ? 1 : 0)) {
            for (int base = lo; base < hi; base += INV_STAGE) {
                const int n = min(INV_STAGE, hi - base);
                __syncthreads();
                if (t == 0) sm.n_dense = 0;
                __syncthreads();
                if (t < n) {                              // one thread per staged slot: its row, its edge list, is it in the band in this tile?
                    const int32_t sl = a.wl.slots[base + t];
                    const uint8_t fl = a.wl.in_tile[(size_t)sl * a.wl.n_tiles + tile];
                    sm.flag[t] = fl;
                    sm.row[t] = a.rows.cur_lo(sl);
                    const int32_t subject = a.slot_subject[sl];
                    sm.mix1[t] = fp_mix1(subject); sm.mix2[t] = fp_mix2(subject);
                    int ne = 0;
                    for (int k = 0; k < a.K; ++k) {
                        const int32_t s2 = a.wl.so_tab[(size_t)sl * SO_STRIDE + k];
                        if (s2 < 0) continue;
                        sm.e_row[t * MAXK + ne] = a.rows.cur_lo(s2);
                        sm.e_so[t * MAXK + ne] = s2; sm.e_k[t * MAXK + ne] = (uint8_t)k;
                        ++ne;
                    }
                    sm.ne[t] = (uint8_t)ne;
                    if (fl) sm.dense[atomicAdd(&sm.n_dense, 1)] = (uint8_t)t;      // (the pass does not depend on the order, SURVEY §7)
                }
                __syncthreads();
                if (!any_k3) continue;
                const int nd = sm.n_dense;
                for (int g = 0; g < nd; g += 4) {
                    // four subjects at a time: their rows and the rows of (up to) two observers each in flight together
                    int idx[4];
                    uint2 w2v[4], e0v[4], e1v[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        idx[q] = g + q < nd ? (int)sm.dense[g + q] : -1;
                        w2v[q] = make_uint2(0xFFFFFFFFu, 0xFFFFFFFFu); e0v[q] = make_uint2(0u, 0u); e1v[q] = make_uint2(0u, 0u);
                        if (idx[q] < 0) continue;
                        w2v[q] = a.rows.load4(sm.row[idx[q]], rb);
                        const int eb = idx[q] * MAXK, ne = sm.ne[idx[q]];
                        if (ne > 0) e0v[q] = a.rows.load4(sm.e_row[eb], rb);
                        if (ne > 1) e1v[q] = a.rows.load4(sm.e_row[eb + 1], rb);
                    }
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int i = idx[q];
                        if (i < 0) continue;
                        const int eb = i * MAXK, ee = eb + sm.ne[i];
                        uint32_t w[4];
#pragma unroll
                        for (int j = 0; j < 4; ++j) w[j] = a.rows.word4(w2v[q], j);
                        uint32_t miss[4];                                   // rings an implicit report could still add, per receiver
                        uint32_t anymiss = 0;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const int c = __popc(w[j] & RM);
                            miss[j] = (k3[j] && c >= a.L && c < a.H) ? (~w[j] & RM) : 0u;   // in this receiver's preProposal
                            anymiss |= miss[j];
                        }
                        if (!anymiss) continue;
                        uint32_t implicit[4] = {0u, 0u, 0u, 0u};
                        for (int ei = eb; ei < ee; ++ei) {
                            const int k = sm.e_k[ei];
                            if (!((anymiss >> k) & 1u)) continue;
                            const uint2 o2 = ei == eb ? e0v[q] : ei == eb + 1 ? e1v[q] : a.rows.load4(sm.e_row[ei], rb);
                            uint32_t wo[4];
#pragma unroll
                            for (int j = 0; j < 4; ++j) wo[j] = a.rows.word4(o2, j);
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                if (!((miss[j] >> k) & 1u)) continue;
                                // observer not in proposal U preProposal.  (No observer here has left in an emitted proposal of an
                                // EARLIER batch: only a receiver that announced holds emit marks, it is frozen from then on, and a
                                // receiver in this pass is active — it had not announced when the batch started.  Its own marks of
                                // this batch are written by phase_mixed_mark, after the pass.)
                                if (__popc(wo[j] & RM) < a.L) continue;
                                // a receiver that already announced explicit proposals in this batch: those subjects left
                                // `proposal` (the transient plane = raised to >= H by this very pass: in the band at entry, not pending)
                                if (MX) {
                                    const int64_t r = rb + j;
                                    if (emitted_in_batch(e, sm.e_so[ei], r, wo[j], splitmix64(a.dl.perm_seed + (uint64_t)(a.rbegin + r)))) continue;
                                }
                                implicit[j] |= 1u << k;
                            }
                        }
                        bool any = false;
                        uint32_t trans = 0;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            if (!implicit[j]) continue;
                            any = true;
                            w[j] |= implicit[j];
                            const bool raised = __popc(w[j] & RM) >= a.H;
                            if (raised && mixed) trans |= 1u << j;             // transient marker, cleared by the unmark phase
                            if (raised) { ++res[j]; kh1[j] += sm.mix1[i]; kh2[j] += sm.mix2[i]; }   // moved preProposal -> proposal
                        }
                        // (the neighbouring thread's 4 receivers share the byte: atomic on the aligned word)
                        if (trans) atomicOr(e.trans.word(a.wl.slots[base + i], rb), trans << (rb & 31));
                        if (any) a.rows.store4(sm.row[i], rb, w);
                    }
                }
            }
        }
        if (P > 1) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (res[j] > 0) { atomicAdd(&e.inv_res[rb + j], res[j]); atomicAdd(&e.inv_h1[rb + j], (unsigned long long)kh1[j]); atomicAdd(&e.inv_h2[rb + j], (unsigned long long)kh2[j]); }
            __threadfence();
            __syncthreads();
            if (t == 0) s_fin = atomicAdd(&e.inv_ticket[tile], 1) == P - 1 ? 1 : 0;
            __syncthreads();
            if (!s_fin) continue;                             // a later block of the tile closes its receivers
            __threadfence();
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                res[j] = atomicExch(&e.inv_res[rb + j], 0);   // (and the accumulators are all zero again)
                kh1[j] = 0; kh2[j] = 0;
                if (res[j] > 0) { kh1[j] = atomicExch(&e.inv_h1[rb + j], 0ull); kh2[j] = atomicExch(&e.inv_h2[rb + j], 0ull); }
            }
            if (t == 0) e.inv_ticket[tile] = 0;
        }
        // ---- finalize2: emissions of the invalidation pass, announced flags --------------------------------------------------
        uint32_t ann = 0;
        bool touched = false;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int64_t r = rb + j;
            if (r >= a.R) continue;
            if (!mine[j] || !(flags[j] & RF_ACTIVE)) { ann |= ((flags[j] & RF_ANNOUNCED) ? 1u : 0u) << (8 * j); continue; }   // not this pass's / settled by finalize1
            touched = true;
            if (res[j] > 0) {
                const int32_t npre = e.n_pre[r] - res[j];
                uint64_t ph1 = e.pend_h1[r] + kh1[j], ph2 = e.pend_h2[r] + kh2[j];
                int32_t pc = e.pend_cnt[r] + res[j];
                if (npre == 0) {
                    // the last unstable subject resolved inside invalidateFailingEdges: proposal (all of it) is emitted
                    e.out_h1[r] += ph1; e.out_h2[r] += ph2; e.out_len[r] += pc;
                    ph1 = 0; ph2 = 0; pc = 0;
                    flags[j] |= RF_ANNOUNCED | RF_ANN_NOW | RF_RULE_GE_H;
                }
                e.n_pre[r] = npre;
                e.pend_h1[r] = ph1; e.pend_h2[r] = ph2; e.pend_cnt[r] = pc;
            }
            flags[j] &= ~RF_K3;
            if ((flags[j] & RF_MIXED_EMIT) && (flags[j] & RF_ANN_NOW) && !(flags[j] & RF_RULE_GE_H)) ++my_inval;   // needs emit marks
            ann |= ((flags[j] & RF_ANNOUNCED) ? 1u : 0u) << (8 * j);
        }
        if (touched) {
            *reinterpret_cast<uint4*>(e.rflags + rb) = make_uint4(flags[0], flags[1], flags[2], flags[3]);
            *reinterpret_cast<uint32_t*>(e.out_ann + rb) = ann;
        }
    }
    if (MX) {
        const int32_t b = block_sum_i32(my_inval, s_red);
        if (t == 0 && b) atomicAdd(&e.bc->n_inval, b);
    }
}

// RF_MIXED_EMIT receivers whose invalidation pass did not emit announce only the explicit part: record it in the emit plane so
// that rapid_cd_get_proposal can list it later (the pre-batch rows are gone by then).  Every slot < S of such a receiver gets its
// bit written, set or clear (the plane is never cleared, see k_gather_proposal).  A warp owns 32 consecutive receivers, i.e. one
// word per slot: lane 0 merges the warp's ballot under the mask of its marked lanes, and nothing else writes that word in the pass.
__device__ __noinline__ void phase_mixed_mark(const ResolveArgs& e, int32_t S) {
    static_assert(GEN_THREADS % 32 == 0, "a warp owns one word of the plane");
    const ApplyArgs& a = e.ap;
    const int spb = 64;
    const int rblocks = (int)(a.Rpad / GEN_THREADS), sblocks = (S + spb - 1) / spb;
    const int64_t items = (int64_t)rblocks * sblocks;
    for (int64_t wi = blockIdx.x; wi < items; wi += gridDim.x) {
        const int64_t r = (wi % rblocks) * GEN_THREADS + threadIdx.x;
        const uint32_t f = r < a.R ? e.rflags[r] : 0u;
        const bool marked = (f & RF_MIXED_EMIT) && (f & RF_ANN_NOW) && !(f & RF_RULE_GE_H);
        const uint32_t mm = __ballot_sync(0xffffffffu, marked);
        if (mm == 0) continue;                                          // (warp-uniform)
        const uint64_t rs = splitmix64(a.dl.perm_seed + (uint64_t)(a.rbegin + r));
        const int32_t s0 = (int32_t)(wi / rblocks) * spb, s1 = min(S, s0 + spb);
        for (int32_t s = s0; s < s1; ++s) {
            const bool em = marked && emitted_in_batch(e, s, r, a.rows.get(s, r), rs);
            const uint32_t b = __ballot_sync(0xffffffffu, em);
            if ((threadIdx.x & 31) == 0) {
                uint32_t* p = e.emit.word(s, r);
                *p = (*p & ~mm) | b;
            }
        }
    }
}

// the transient plane back to all zero: 128 bytes per listed (subject, tile) pair, the only places the pass can have set bits
__device__ void phase_inval_unmark(const ResolveArgs& e) {
    const ApplyArgs& a = e.ap;
    const int n_list = min(*(volatile int32_t*)a.wl.count, a.wl.cap);
    constexpr int TW = TILE_R / 32;                                     // words of a tile
    const int64_t items = (int64_t)n_list * a.wl.n_tiles * TW;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < items; q += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = q / TW;
        const int32_t sl = a.wl.slots[p / a.wl.n_tiles];
        const int tile = (int)(p % a.wl.n_tiles);
        if (!a.wl.in_tile[(size_t)sl * a.wl.n_tiles + tile]) continue;
        e.trans.p[(size_t)sl * e.trans.words + (size_t)tile * TW + (size_t)(q % TW)] = 0u;
    }
}

// the last block to get here copies the counters for the host and re-arms the per-batch fields for the next batch
__device__ void resolve_tail(const ResolveArgs& a, int32_t serial) {
    __shared__ int s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = atomicAdd(&a.bc->ticket, 1) == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last || threadIdx.x != 0) return;
    __threadfence();
    volatile BatchCounts* b = a.bc;
    BatchCounts c;
    c.n_slots = b->n_slots; c.n_valid = b->n_valid; c.n_batch_subj = b->n_batch_subj; c.any_down = b->any_down;
    c.bad_ring = b->bad_ring; c.bad_dst = b->bad_dst; c.n_mixed = b->n_mixed; c.n_inval = b->n_inval; c.S_before = b->S_before;
    c.overflow = b->overflow; c.need_slots = b->need_slots; c.n_times = b->n_times; c.mixed_iters = b->mixed_iters;
    c.n_pairs = *(volatile int32_t*)a.ap.wl.count; c.ticket = 0; c.serial = serial;
    c.seq_last = b->seq_last; c.seq_down = b->seq_down; c.seq_abort = b->seq_abort; c.seq_a1 = b->seq_a1; c.seq_a2 = b->seq_a2;
    c.mx_first = b->mx_first; c.mx_left = b->mx_left;
    if (c.seq_abort) { c.n_slots = c.S_before; b->n_slots = c.S_before; }   // the slots this call assigned were given back (seq_rollback)
    // errors stay latched until the host has collected them (an asynchronous caller may have several batches in flight)
    c.sticky_bad_ring = b->sticky_bad_ring | (c.bad_ring >= 0 ? 1 : 0);
    c.sticky_bad_dst = b->sticky_bad_dst | (c.bad_dst >= 0 ? 1 : 0);
    c.sticky_overflow = b->sticky_overflow | (c.overflow ? 1 : 0);
    b->sticky_bad_ring = c.sticky_bad_ring; b->sticky_bad_dst = c.sticky_bad_dst; b->sticky_overflow = c.sticky_overflow;
    *a.snap = c;
    b->n_valid = 0; b->n_batch_subj = 0; b->any_down = 0; b->bad_ring = -1; b->bad_dst = -1; b->n_mixed = 0; b->n_inval = 0;
    b->overflow = 0; b->need_slots = 0; b->n_times = 0; b->mixed_iters = 0; b->ticket = 0;
    b->seq_last = 0; b->seq_down = INT_MAX; b->seq_abort = 0; b->seq_a1 = 0; b->seq_a2 = 0; b->mx_first = INT_MAX; b->mx_left = 0;
    b->S_before = c.n_slots;                                            // the next batch starts from here (k_prepare reads it)
}

// ---- the reference-receiver shortcut of the interval analysis (uniform delivery) ------------------------------------------------------
// mx_dev: one bit per receiver, set if it differs from receiver r0 in the pre-batch word of SOME batch subject
__device__ void phase_ref_compare(const ResolveArgs& e, const int64_t r0, const int Sb, const int S_before) {
    static_assert(TILE_R == 4 * GEN_THREADS, "a thread owns 4 receivers of a tile");
    const ApplyArgs& a = e.ap;
    const uint32_t RM = (1u << a.K) - 1u;
    const int t = threadIdx.x;
    // work items: (tile, chunk of subjects); a block-wide OR-reduction is not needed — each thread owns its 4 receivers' bits
    constexpr int CH = 64;
    __shared__ const uint8_t* s_row[CH];
    __shared__ uint32_t s_ref[CH];
    const int nch = (Sb + CH - 1) / CH;
    const int64_t items = (int64_t)a.n_tiles * nch;
    for (int64_t wi = blockIdx.x; wi < items; wi += gridDim.x) {
        const int tile = (int)(wi % a.n_tiles), ch = (int)(wi / a.n_tiles);
        const int64_t rb = (int64_t)tile * TILE_R + (int64_t)t * 4;
        const int b0 = ch * CH, nb = min(Sb, b0 + CH) - b0;
        __syncthreads();
        if (t < nb) {
            const int32_t slot = a.desc[b0 + t].slot;
            const uint8_t* row = slot >= S_before ? nullptr : a.rows.cur_lo(slot);   // pre-batch row (not flipped yet); fresh: state 0 for everyone
            s_row[t] = row;
            s_ref[t] = row ? a.rows.get(row, r0) & RM : 0u;
        }
        __syncthreads();
        uint32_t bits = 0;
#pragma unroll 8
        for (int i = 0; i < nb; ++i) {
            const uint8_t* row = s_row[i];
            if (row == nullptr) continue;
            const uint2 g = a.rows.load4(row, rb);
#pragma unroll
            for (int j = 0; j < 4; ++j) bits |= ((a.rows.word4(g, j) ^ s_ref[i]) & RM) ? 1u << j : 0u;
        }
        if (bits) atomicOr(&e.mx_dev[rb >> 5], bits << (rb & 31));
    }
}
// the flagged receivers that agree with r0 take its outcome; the others are counted (bc->mx_left) and go through the general passes
__device__ void phase_ref_adopt(const ResolveArgs& a, const int64_t r0, int32_t* s_red) {
    const uint32_t f0 = a.mx_fl[r0];
    int32_t my = 0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.ap.R; r += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t fl = a.mx_fl[r];
        const bool dev = (a.mx_dev[r >> 5] >> (r & 31)) & 1u;
        if (r != r0 && (fl & MX_ON) && !(fl & MX_DONE)) {
            if (!dev) {
                a.mx_fl[r] = f0 ? (f0 | MX_REF) : 0u;                           // 0: nothing was emitted explicitly
                if ((f0 & MX_DONE) && (f0 & MX_HAS_E)) { a.estar[r] = a.estar[r0]; a.mx_e1[r] = a.mx_e1[r0]; a.mx_e2[r] = a.mx_e2[r0]; a.mx_ec[r] = a.mx_ec[r0]; }
            } else {
                ++my;
            }
        }
    }
    const int32_t b = block_sum_i32(my, s_red);
    if (threadIdx.x == 0 && b) atomicAdd(&a.bc->mx_left, b);
    if (blockIdx.x == 0 && threadIdx.x == 0 && f0) a.mx_fl[r0] = f0 | MX_REF;
}

// ==================================================================================================================
// k_seq_check: the two premises of the one-pass treatment of a sequence of batches (see visit_prefix), per receiver.
// blockIdx.y == 0: A1 from the partial accumulators; blockIdx.y >= 1: A2 over a chunk of the dictionary's slots.  Counts
// the receivers that fail into bc->seq_abort — every later kernel of the batch returns at once if that is non-zero.
// ==================================================================================================================
__global__ void __launch_bounds__(GEN_THREADS) k_seq_check(const ResolveArgs* __restrict__ ga) {
    const ResolveArgs& a = *ga;
    const ApplyArgs& ap = a.ap;
    __shared__ int32_t s_red[GEN_THREADS / 32];
    __shared__ ChunkAcc s_fresh;
    __shared__ int s_fhave;
    if (a.bc->overflow) return;
    const int64_t r = (int64_t)blockIdx.x * GEN_THREADS + threadIdx.x;
    const uint32_t rf = r < ap.R ? a.rflags[r] : RF_ANNOUNCED;
    const bool active = r < ap.R && !(rf & RF_ANNOUNCED) && !((ap.dl.flags & RAPID_DELIVERY_BLOCKED) && ap.dl.blocked[r]);
    int32_t bad = 0;
    if (blockIdx.y == 0) {
        // ---- A1: no proposal can have been emitted before the last batch ------------------------------------------------------
        reduce_fresh(a, &s_fresh, &s_fhave);
        if (active) {
            uint32_t tpc = s_fresh.tpc, mBH = s_fresh.minBHp, mBL = s_fresh.minBLlong;
            const int tile = (int)(r / TILE_R);
            for (int c = 0; c < a.n_chunks; ++c) {
                if (!ap.part.flag[(size_t)c * ap.part.n_tiles + tile]) continue;
                const size_t p = (size_t)c * ap.Rpad + (size_t)r;
                tpc += ap.part.cntp[p].z;
                const uint2 q = ap.part.seq[p];
                mBH = min(mBH, q.x); mBL = min(mBL, q.y);
            }
            // an H-crossing in the prefix needs a subject that sits in the band from an EARLIER batch (or an untouched one
            // that has been there since before the call) until the last batch starts
            const bool ok = mBH == T32_NONE || (a.n_pre[r] - (int32_t)tpc) > 0 || mBL < mBH;
            if (!ok) bad = 1;
        }
    } else {
        // ---- A2: no invalidation pass at the end of a prefix batch reports a ring of a subject the call does NOT touch ------------
        // (the subjects the call touches carry their implicit reports through the visit: prefix_core)
        const int32_t S = a.bc->n_slots, S_before = a.bc->S_before;
        const uint32_t last = (uint32_t)a.bc->seq_last;                   // prefix batches are 1 .. last (1-based)
        const int nchunks = (int)gridDim.y - 1;
        const int per = (S + nchunks - 1) / nchunks;
        const int32_t q0 = min(S, ((int)blockIdx.y - 1) * per), q1 = min(S, q0 + per);
        const uint32_t RM = (1u << ap.K) - 1u;
        const uint32_t bDown = receiver_down_batch(ap, rf, false);
        for (int32_t sl = q0; sl < q1; ++sl) {
            if (sl >= S_before || !ap.wl.has_so[sl] || a.touch[sl] == a.serial) continue;      // (uniform across the block)
            if (!active || bDown == T32_NONE) continue;
            const uint32_t us = ap.rows.get(sl, r) & RM;
            const int cs = __popc(us);
            if (cs < ap.L || cs >= ap.H) continue;                         // not in this receiver's preProposal
            for (int k = 0; k < ap.K; ++k) {
                const int32_t so = ap.wl.so_tab[(size_t)sl * SO_STRIDE + k];
                if (so < 0 || ((us >> k) & 1u)) continue;
                const bool o_touched = a.touch[so] == a.serial;
                const int bo_idx = o_touched ? a.batch_index[so] : 0;
                const uint32_t uo = so < S_before ? (ap.rows.get(so, r) & RM) : 0u;
                const uint32_t bLo = observer_L_batch(uo, o_touched ? &ap.desc[bo_idx] : nullptr, o_touched ? &ap.pwalk[bo_idx] : nullptr, ap.L);
                if (bLo != T32_NONE && max(bLo, bDown) <= last) bad = 1;  // an invalidation pass inside the prefix would report ring k
            }
        }
    }
    const int32_t b = block_sum_i32(bad, s_red);
    if (threadIdx.x == 0 && b) { atomicAdd(&a.bc->seq_abort, b); atomicAdd(blockIdx.y == 0 ? &a.bc->seq_a1 : &a.bc->seq_a2, b); }
}

// ---- the four launches after the apply kernel (no host round trip between them) ---------------------------------------------
__global__ void __launch_bounds__(GEN_THREADS) k_finalize1(const ResolveArgs* __restrict__ ga) {
    const ResolveArgs& a = *ga;
    __shared__ int32_t s_red[GEN_THREADS / 32];
    if (a.bc->overflow || a.bc->seq_abort) return;                      // rolled back by k_prepare / the sequence is replayed batch by batch
    phase_finalize1(a, s_red);
}

// cooperative, ALWAYS launched: with nothing flagged it just flips the rows (a few microseconds)
__global__ void __launch_bounds__(GEN_THREADS, 2) k_mixed_flip(const ResolveArgs* __restrict__ ga) {
    const ResolveArgs& a = *ga;
    cg::grid_group grid = cg::this_grid();
    __shared__ PassSmem sm;
    __shared__ int32_t s_red[GEN_THREADS / 32];
    if (a.bc->overflow || a.bc->seq_abort) return;                      // (no flip: the pre-call rows stay current)
    const int Sb = a.bc->n_batch_subj, S_before = a.bc->S_before;
    if (a.counts_only && a.bc->n_times > 0 && Sb > 0) {
        mixed_pass<2>(a, sm, Sb, S_before);
        grid.sync();
        phase_classify_moments(a, s_red);
        grid.sync();
    }
    const int mixed = *(volatile int32_t*)&a.bc->n_mixed > 0 ? 1 : 0;
    if (mixed && Sb > 0) {
        auto analyse = [&](const int64_t only_r) -> int {       // the fixpoint loop + the sum pass, for everyone flagged or for one receiver
            int it = 0;
            for (;; ++it) {
                mixed_pass<0>(a, sm, Sb, S_before, only_r);
                grid.sync();
                if (blockIdx.x == 0 && threadIdx.x == 0) a.mx_changed[(it + 2) & 3] = 0;
                phase_mixed_update(a, &a.mx_changed[it & 3], s_red, only_r);
                grid.sync();
                if (*(volatile int32_t*)&a.mx_changed[it & 3] == 0 || it > Sb + 1) break;
            }
            mixed_pass<1>(a, sm, Sb, S_before, only_r);
            grid.sync();
            if (blockIdx.x == 0 && threadIdx.x == 0) { a.mx_changed[0] = 0; a.mx_changed[1] = 0; a.mx_changed[2] = 0; a.mx_changed[3] = 0; }
            grid.sync();
            return it + 1;
        };
        int iters = 0;
        int left = 1;
        if (a.uniform && !a.ap.seq) {
            // Uniform delivery: receivers that hold the same words for the batch's subjects get the same intervals, hence the same
            // answer.  Analyse ONE flagged receiver, find the flagged receivers that agree with it on every batch subject (one
            // read-only pass over the pre-batch rows) and hand them its result; only the others take the passes below.
            const int64_t r0 = (int64_t)*(volatile int32_t*)&a.bc->mx_first;
            iters = analyse(r0);
            phase_ref_compare(a, r0, Sb, S_before);
            grid.sync();
            phase_ref_adopt(a, r0, s_red);
            grid.sync();
            left = *(volatile int32_t*)&a.bc->mx_left;
            // (every block is past the adoption: the difference bits go back to all-zero for the next batch)
            for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < (int64_t)(a.ap.Rpad >> 5); q += (int64_t)gridDim.x * blockDim.x) a.mx_dev[q] = 0;
        }
        if (left > 0) iters += analyse(-1);
        if (blockIdx.x == 0 && threadIdx.x == 0) a.bc->mixed_iters = iters;
        phase_mixed_commit(a);
        grid.sync();
    }
    // flip: the rows the apply kernel wrote become current (the interval analysis above still needed the pre-batch rows)
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < Sb; b += gridDim.x * blockDim.x) a.cur_w[a.ap.desc[b].slot] ^= 1;
}

__global__ void __launch_bounds__(GEN_THREADS, 2) k_inval_finalize2(const ResolveArgs* __restrict__ ga) {
    const ResolveArgs& a = *ga;
    __shared__ InvSmem sm;
    __shared__ int32_t s_red[GEN_THREADS / 32];
    const int mixed = a.bc->n_mixed > 0 ? 1 : 0;
    if (!a.bc->overflow && !a.bc->seq_abort) phase_inval_finalize2<false>(a, mixed, sm, s_red);
    if (a.bc->seq_abort) {
        // the one-pass treatment of the sequence was refused: give back the slots this call assigned (their rows were written
        // but never made current), so that the batch-by-batch replay sees the dictionary of before the call
        const int32_t s0 = a.bc->S_before, s1 = a.bc->n_slots;
        for (int32_t sl = s0 + blockIdx.x * blockDim.x + threadIdx.x; sl < s1; sl += gridDim.x * blockDim.x)
            const_cast<int32_t*>(a.slot_of)[a.ap.slot_subject[sl]] = -1;
    }
    if (!mixed) resolve_tail(a, a.serial);                               // else k_marks closes the batch
}

// cooperative, ALWAYS launched: returns at once unless some receiver went through the interval analysis
__global__ void __launch_bounds__(GEN_THREADS, 2) k_marks(const ResolveArgs* __restrict__ ga) {
    const ResolveArgs& a = *ga;
    cg::grid_group grid = cg::this_grid();
    __shared__ InvSmem sm;
    __shared__ int32_t s_red[GEN_THREADS / 32];
    if (a.bc->n_mixed <= 0) return;                                      // (k_inval_finalize2 closed the batch)
    phase_inval_finalize2<true>(a, 1, sm, s_red);                        // the receivers k_inval_finalize2 left out
    grid.sync();
    if (*(volatile int32_t*)&a.bc->n_inval > 0) {
        // receivers that announce only the explicit part: persist it in the emit plane while the pre-batch rows still exist
        phase_mixed_mark(a, *(volatile int32_t*)&a.bc->n_slots);
        grid.sync();
    }
    phase_inval_unmark(a);                                              // only now: the marks above still needed the transient plane
    resolve_tail(a, a.serial);
}

// ------------------------------------------------------------------------------------------------------------------
// host orchestration
// ------------------------------------------------------------------------------------------------------------------
static Bucketed* state(CD* cd) {
    if (!cd->bucketed_state) cd->bucketed_state = new Bucketed();
    return static_cast<Bucketed*>(cd->bucketed_state);
}

void bucketed_destroy(CD* cd) {
    if (cd->bucketed_state) { delete static_cast<Bucketed*>(cd->bucketed_state); cd->bucketed_state = nullptr; }
}

static WorkList worklist(const Bucketed* b) {
    WorkList wl;
    wl.has_so = b->has_so.p; wl.so_tab = b->wl_so_tab.p; wl.in_tile = b->wl_in_tile.p; wl.listed = b->wl_listed.p;
    wl.slots = b->wl_slots.p; wl.count = b->wl_count.p;
    wl.cap = (int32_t)std::min<size_t>(b->in_list_slots, 0x7fffffff); wl.n_tiles = b->n_tiles;
    return wl;
}

// the work-list arrays follow the handle's slot capacity (they only ever grow, with the contents kept)
template <typename T>
static int32_t grow_keep(DevBuf<T>& buf, size_t n_old, size_t n_new, cudaStream_t s) {
    DevBuf<T> nb;
    RAPID_CHECK(nb.reserve(std::max<size_t>(n_new, 1)));
    RAPID_CUDA(cudaMemsetAsync(nb.p, 0, std::max<size_t>(n_new, 1) * sizeof(T), s));
    if (n_old && buf.p) RAPID_CUDA(cudaMemcpyAsync(nb.p, buf.p, n_old * sizeof(T), cudaMemcpyDeviceToDevice, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    std::swap(buf.p, nb.p); std::swap(buf.cap, nb.cap);
    return RAPID_OK;
}

static int32_t ensure_pre_capacity(CD* cd, Bucketed* b) {
    const size_t slots = cd->S_cap;
    if (slots <= b->in_list_slots) return RAPID_OK;
    const size_t o = b->in_list_slots, nt = (size_t)b->n_tiles;
    RAPID_CHECK(grow_keep(b->wl_in_tile, o * nt, slots * nt, cd->stream));
    RAPID_CHECK(grow_keep(b->wl_listed, o, slots, cd->stream));
    RAPID_CHECK(grow_keep(b->wl_slots, o, slots, cd->stream));
    RAPID_CHECK(grow_keep(b->wl_so_tab, o * SO_STRIDE, slots * SO_STRIDE, cd->stream));
    RAPID_CHECK(grow_keep(b->has_so, o, slots, cd->stream));
    b->in_list_slots = slots;
    return RAPID_OK;
}

int32_t bucketed_prep_buffers(CD* cd, int64_t A, PrepOut* po) {
    Bucketed* b = state(cd);
    b->n_tiles = (int)(cd->Rpad / TILE_R);
    RAPID_CHECK(ensure_pre_capacity(cd, b));
    const size_t a = (size_t)std::max<int64_t>(A, 1);
    RAPID_CHECK(b->desc.reserve(a)); RAPID_CHECK(b->walk.reserve(a)); RAPID_CHECK(b->pwalk.reserve(a));
    RAPID_CHECK(b->sidx.reserve(a)); RAPID_CHECK(b->s_ring.reserve(a)); RAPID_CHECK(b->s_status.reserve(a));
    // per-slot scratch: a batch can touch at most S_cap slots (a batch that needs more is rolled back on the device)
    const size_t slots = std::max<size_t>(cd->S_cap, 1);
    RAPID_CHECK(b->batch_index.reserve(slots));
    RAPID_CHECK(b->batch_slots.reserve(slots));
    RAPID_CHECK(b->bins.reserve(slots * 64));
    RAPID_CHECK(b->ovf.reserve(a)); RAPID_CHECK(b->cell_batch.reserve(a));
    if (slots > b->seg_cnt.cap) {
        RAPID_CHECK(b->seg_cnt.reserve(slots));
        RAPID_CUDA(cudaMemsetAsync(b->seg_cnt.p, 0, b->seg_cnt.cap * sizeof(int32_t), cd->stream));
    }
    po->desc = b->desc.p; po->walk = b->walk.p; po->sidx = b->sidx.p; po->s_ring = b->s_ring.p; po->s_status = b->s_status.p;
    po->batch_index = b->batch_index.p; po->seg_cnt = b->seg_cnt.p; po->batch_slots = b->batch_slots.p;
    po->bins = b->bins.p; po->ovf = b->ovf.p; po->pwalk = b->pwalk.p; po->cell_batch = b->cell_batch.p;
    po->wl = worklist(b);
    return RAPID_OK;
}

__global__ void k_clear_sticky(BatchCounts* bc) { bc->sticky_bad_ring = 0; bc->sticky_bad_dst = 0; bc->sticky_overflow = 0; }

int32_t bucketed_clear_sticky(CD* cd) {
    k_clear_sticky<<<1, 1, 0, cd->stream>>>(cd->counts.p);
    RAPID_KERNEL_CHECK();
    return RAPID_OK;
}

// clear() of a bucketed handle in ONE launch: every receiver's detector scalars (MultiNodeCutDetector.java:169-178 +
// announcedProposal = false), the subject dictionary (O(#slots in use)), the invalidation work list, and — by the last block to
// finish, because the loops above read the slot count and the list length — the device counters for a new configuration epoch.
struct ClearArgs {
    int64_t Rpad;
    int32_t* n_pre; int32_t* n_prop; uint32_t* rflags;
    uint64_t* pend_h1; uint64_t* pend_h2; int32_t* pend_cnt;
    uint64_t* out_h1; uint64_t* out_h2; int32_t* out_len; uint8_t* out_ann;
    BatchCounts* bc; BatchCounts* snap;
    const int32_t* slot_subject; int32_t* slot_of; uint8_t* cur;
    WorkList wl;
    int has_wl;
};
__global__ void __launch_bounds__(256) k_clear_bucketed(const ClearArgs a) {
    __shared__ int s_last;
    const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, gthreads = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = gtid; r < a.Rpad; r += gthreads) {
        a.n_pre[r] = 0; a.n_prop[r] = 0; a.rflags[r] = 0u;
        a.pend_h1[r] = 0; a.pend_h2[r] = 0; a.pend_cnt[r] = 0;
        a.out_h1[r] = 0; a.out_h2[r] = 0; a.out_len[r] = 0; a.out_ann[r] = 0;
    }
    const int32_t S = a.bc->n_slots;
    for (int64_t sl = gtid; sl < S; sl += gthreads) { a.slot_of[a.slot_subject[sl]] = -1; a.cur[sl] = 0; }
    if (a.has_wl) {
        const int n = min(*a.wl.count, a.wl.cap);
        const int64_t items = (int64_t)n * a.wl.n_tiles;
        for (int64_t e = gtid; e < items; e += gthreads) {
            const int32_t sl = a.wl.slots[e / a.wl.n_tiles];
            const int tile = (int)(e % a.wl.n_tiles);
            a.wl.in_tile[(size_t)sl * a.wl.n_tiles + tile] = 0;
            if (tile == 0) a.wl.listed[sl] = 0;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = atomicAdd(&a.bc->ticket, 1) == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last || threadIdx.x != 0) return;
    __threadfence();
    BatchCounts c;
    memset(&c, 0, sizeof(c));
    c.bad_ring = -1; c.bad_dst = -1; c.seq_down = INT_MAX; c.mx_first = INT_MAX;
    volatile BatchCounts* b = a.bc;
    c.sticky_bad_ring = b->sticky_bad_ring; c.sticky_bad_dst = b->sticky_bad_dst; c.sticky_overflow = b->sticky_overflow;   // errors not collected yet survive a clear()
    *a.bc = c;
    *a.snap = c;
    *a.wl.count = 0;
}

int32_t bucketed_clear(CD* cd) {
    if (!cd->bucketed) return RAPID_OK;
    Bucketed* b = state(cd);
    b->n_tiles = (int)(cd->Rpad / TILE_R);
    cudaStream_t s = cd->stream;
    if (!b->wl_count.p) {
        RAPID_CHECK(b->wl_count.reserve(1));
        RAPID_CUDA(cudaMemsetAsync(b->wl_count.p, 0, sizeof(int32_t), s));
        RAPID_CHECK(b->mx_changed.reserve(4));
        RAPID_CUDA(cudaMemsetAsync(b->mx_changed.p, 0, 4 * sizeof(int32_t), s));
    }
    ClearArgs a;
    a.Rpad = (int64_t)cd->Rpad;
    a.n_pre = cd->n_pre.p; a.n_prop = cd->n_prop.p; a.rflags = cd->rflags.p;
    a.pend_h1 = cd->pend_h1.p; a.pend_h2 = cd->pend_h2.p; a.pend_cnt = cd->pend_cnt.p;
    a.out_h1 = cd->out_h1.p; a.out_h2 = cd->out_h2.p; a.out_len = cd->out_len.p; a.out_ann = cd->out_ann.p;
    a.bc = cd->counts.p; a.snap = cd->counts_snap.p;
    a.slot_subject = cd->slot_subject.p; a.slot_of = cd->slot_of.p; a.cur = cd->cur.p;
    a.wl = worklist(b); a.has_wl = b->in_list_slots ? 1 : 0;
    const unsigned grid = (unsigned)std::max<size_t>(1, std::min<size_t>(ceil_div<size_t>(cd->Rpad, 256), (size_t)TARGET_SMS * 8));
    k_clear_bucketed<<<grid, 256, 0, s>>>(a);
    RAPID_KERNEL_CHECK();
    return RAPID_OK;
}

template <int HB>
static void launch_uniform(dim3 grid, cudaStream_t s, const ApplyArgs& ap, bool counts_only, bool seq) {
    if (seq) {
        if (counts_only) k_apply_uniform<true, true, HB><<<grid, UNI_THREADS, 0, s>>>(ap);
        else k_apply_uniform<false, true, HB><<<grid, UNI_THREADS, 0, s>>>(ap);
    } else {
        if (counts_only) k_apply_uniform<true, false, HB><<<grid, UNI_THREADS, 0, s>>>(ap);
        else k_apply_uniform<false, false, HB><<<grid, UNI_THREADS, 0, s>>>(ap);
    }
}

// Everything of one batch after k_prepare, enqueued on the handle's stream with NO host synchronisation: the apply kernel
// (grid sized from an ESTIMATE of the number of batch subjects — the kernels take the real one from the device counters), the
// cooperative resolve kernel, and the copy of the counter snapshot to pinned host memory.
int32_t bucketed_apply(CD* cd, int64_t A, const DeliveryDev& dl, bool seq) {
    Bucketed* b = state(cd);
    cudaStream_t s = cd->stream;
    const bool uniform = !(dl.flags & (RAPID_DELIVERY_BITMAP | RAPID_DELIVERY_PERMUTED));
    const bool counts_only = (dl.flags & RAPID_DELIVERY_PERMUTED) && !(dl.flags & RAPID_DELIVERY_BITMAP);
    const bool swar = uniform || counts_only;          // k_apply_uniform<PERM>: 8 receivers per thread
    b->n_tiles = (int)(cd->Rpad / TILE_R);

    if (b->slots_uniform == 0) {
        int dev = 0, sms = TARGET_SMS, per_u = 8, per_g = 4, per_r = 2;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_u, k_apply_uniform<false, false, 2>, UNI_THREADS, 0);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_g, k_apply_generic, GEN_THREADS, 0);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_r, k_mixed_flip, GEN_THREADS, 0);
        int per_m = 2;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_m, k_marks, GEN_THREADS, 0);
        per_r = std::min(per_r, per_m);
        b->slots_uniform = sms * std::max(per_u, 1);
        b->slots_generic = sms * std::max(per_g, 1);
        b->resolve_grid = sms * std::max(per_r, 1);
    }
    // ---- grid: tiles x subject chunks, a few waves of the SMs ---------------------------------------------------------
    // The number of batch subjects is only known on the device; the previous batch's ratio of subjects to cells (or one
    // subject per K/2 cells) is a good enough guess — it only shapes the grid, the kernels split the real count.
    int Sb = (int)std::max<int64_t>(1, std::min<int64_t>(A, cd->est_A > 0 ? (A * (int64_t)std::max(cd->est_Sb, 1) + cd->est_A - 1) / cd->est_A
                                                                           : (2 * A + cd->K - 1) / cd->K));
    Sb = (int)std::min<int64_t>(Sb, (int64_t)std::max<size_t>(cd->S_cap, 1));
    int n_chunks = 1;
    {
        const int rblocks = swar ? b->n_tiles : (int)(cd->Rpad / GEN_THREADS);
        // Pick the number of subject chunks so that (tiles x chunks) blocks fill whole waves of resident blocks:
        // a bandwidth-bound grid whose last wave is mostly empty pays almost a full wave for it.  More chunks also
        // mean more per-receiver partials (48 B each), so cap them at ~8 % of the mask traffic.
        const int slots = swar ? b->slots_uniform : b->slots_generic;
        const int cmax = std::max(1, std::min(Sb, std::max(Sb / 300, ceil_div(slots, rblocks))));
        double best = -1.0;
        for (int c = 1; c <= cmax; ++c) {
            const int ch = ceil_div(Sb, c), cc = ceil_div(Sb, ch);
            // cost model (a heuristic; RAPID_B200_CHUNKS overrides it): the share of HBM bandwidth a grid of w waves of resident
            // blocks reaches
            const double w = (double)rblocks * cc / slots;
            const double f = w - std::floor(w);
            double eff;
            if (w <= 1.0) eff = 0.85 + 0.15 * w;                                   // one partial wave: a little less occupancy
            else eff = w / (std::floor(w) + (f > 0 ? std::max(f, 0.6) : 0.0));     // tail wave: needs ~60 % of the slots to saturate HBM
            eff -= 0.001 * cc;                                                     // per-chunk prologue (fresh subjects cost no partials)
            if (eff > best) { best = eff; n_chunks = cc; }
        }
        if (const char* ov = getenv("RAPID_B200_CHUNKS")) n_chunks = std::max(1, std::min(Sb, atoi(ov)));   // test hook: forced chunk counts
    }
    cd->last_chunks = n_chunks;
    const size_t pn = (size_t)n_chunks * cd->Rpad;
    RAPID_CHECK(b->p_cnt.reserve(pn)); RAPID_CHECK(b->p_minTH.reserve(pn)); RAPID_CHECK(b->p_minTLun.reserve(pn));
    RAPID_CHECK(b->p_h1.reserve(pn)); RAPID_CHECK(b->p_h2.reserve(pn));
    if (seq) {
        RAPID_CHECK(b->p_cntp.reserve(pn)); RAPID_CHECK(b->p_h1p.reserve(pn)); RAPID_CHECK(b->p_h2p.reserve(pn));
        RAPID_CHECK(b->p_seq.reserve(pn));
    }
    RAPID_CHECK(b->mx_fl.reserve(cd->Rpad)); RAPID_CHECK(b->mx_a.reserve(cd->Rpad)); RAPID_CHECK(b->mx_cand.reserve(cd->Rpad));
    RAPID_CHECK(b->mx_emax.reserve(cd->Rpad)); RAPID_CHECK(b->mx_p1.reserve(cd->Rpad)); RAPID_CHECK(b->mx_p2.reserve(cd->Rpad));
    RAPID_CHECK(b->mx_pc.reserve(cd->Rpad)); RAPID_CHECK(b->estar.reserve(cd->Rpad));
    if (!b->mx_dev.p || b->mx_dev.cap < (cd->Rpad >> 5)) {
        RAPID_CHECK(b->mx_dev.reserve(std::max<size_t>(cd->Rpad >> 5, 1)));
        RAPID_CUDA(cudaMemsetAsync(b->mx_dev.p, 0, std::max<size_t>(cd->Rpad >> 5, 1) * sizeof(uint32_t), s));
    }
    if (!b->mx_e1.p) {
        RAPID_CHECK(b->mx_e1.reserve(cd->Rpad)); RAPID_CHECK(b->mx_e2.reserve(cd->Rpad)); RAPID_CHECK(b->mx_ec.reserve(cd->Rpad));
        RAPID_CUDA(cudaMemsetAsync(b->mx_e1.p, 0, cd->Rpad * sizeof(unsigned long long), s));
        RAPID_CUDA(cudaMemsetAsync(b->mx_e2.p, 0, cd->Rpad * sizeof(unsigned long long), s));
        RAPID_CUDA(cudaMemsetAsync(b->mx_ec.p, 0, cd->Rpad * sizeof(int32_t), s));
    }
    RAPID_CHECK(b->p_flag.reserve((size_t)n_chunks * std::max(b->n_tiles, 1)));
    RAPID_CHECK(b->p_chunk.reserve((size_t)n_chunks));
    Partials part{b->p_cnt.p, b->p_cntp.p, b->p_minTH.p, b->p_minTLun.p, b->p_h1.p, b->p_h2.p, b->p_h1p.p, b->p_h2p.p, b->p_seq.p, b->p_flag.p, b->p_chunk.p, b->n_tiles};

    ApplyArgs ap;
    ap.rows = RowRef{cd->masks.p, cd->cur.p, cd->Rpad, cd->row_stride, cd->nbuf, cd->hb}; ap.Rpad = cd->Rpad;
    ap.K = cd->K; ap.H = cd->H; ap.L = cd->L; ap.R = cd->R; ap.rbegin = cd->rbegin;
    ap.rflags = cd->rflags.p; ap.dl = dl; ap.bc = cd->counts.p;
    ap.desc = b->desc.p; ap.walk = b->walk.p; ap.pwalk = b->pwalk.p; ap.slot_subject = cd->slot_subject.p;
    ap.touch = cd->touch.p; ap.batch_index = b->batch_index.p; ap.serial = cd->batch_serial; ap.seq = seq ? 1 : 0;
    ap.sidx = b->sidx.p; ap.s_ring = b->s_ring.p; ap.s_status = b->s_status.p;
    ap.part = part; ap.n_tiles = b->n_tiles; ap.wl = worklist(b);

    RAPID_CUDA(cudaEventRecord(cd->evk0, s));
    if (swar) {
        dim3 grid((unsigned)b->n_tiles, (unsigned)n_chunks);
        if (cd->hb == 2) launch_uniform<2>(grid, s, ap, counts_only, seq);
        else launch_uniform<8>(grid, s, ap, counts_only, seq);
        cd->last_path = counts_only ? 4 : 2;
    } else {
        dim3 grid((unsigned)(cd->Rpad / GEN_THREADS), (unsigned)n_chunks);
        k_apply_generic<<<grid, GEN_THREADS, 0, s>>>(ap);
        cd->last_path = 3;
    }
    RAPID_KERNEL_CHECK();
    RAPID_CUDA(cudaEventRecord(cd->evk1, s));

    ResolveArgs ra;
    ra.ap = ap; ra.bc = cd->counts.p;
    ra.emit = MarkPlane{cd->emit_marks.p, cd->Rpad / 32}; ra.trans = MarkPlane{cd->trans_marks.p, cd->Rpad / 32}; ra.snap = cd->counts_snap.p; ra.n_chunks = n_chunks;
    ra.uniform = uniform ? 1 : 0; ra.counts_only = counts_only ? 1 : 0; ra.cur_w = cd->cur.p;
    ra.seq = seq ? 1 : 0; ra.seq_dev = nullptr;
    ra.n_pre = cd->n_pre.p; ra.rflags = cd->rflags.p; ra.pend_h1 = cd->pend_h1.p; ra.pend_h2 = cd->pend_h2.p;
    ra.pend_cnt = cd->pend_cnt.p; ra.out_h1 = cd->out_h1.p; ra.out_h2 = cd->out_h2.p; ra.out_len = cd->out_len.p; ra.out_ann = cd->out_ann.p;
    ra.mx_fl = b->mx_fl.p; ra.mx_a = b->mx_a.p; ra.mx_cand = b->mx_cand.p; ra.mx_emax = b->mx_emax.p;
    ra.mx_p1 = b->mx_p1.p; ra.mx_p2 = b->mx_p2.p; ra.mx_pc = b->mx_pc.p; ra.estar = b->estar.p;
    ra.mx_e1 = b->mx_e1.p; ra.mx_e2 = b->mx_e2.p; ra.mx_ec = b->mx_ec.p; ra.mx_changed = b->mx_changed.p; ra.mx_dev = b->mx_dev.p;
    ra.slot_of = cd->slot_of.p; ra.obs = cd->view->obs.p; ra.touch = cd->touch.p; ra.batch_index = b->batch_index.p;
    ra.serial = cd->batch_serial;
    // blocks per tile of the invalidation pass: enough to fill the device twice over when the tiles alone are far from it.
    // A few tiles walked by one block each leave most SMs idle (BASELINE config 3: 10 tiles); from 64 tiles on the tiles alone
    // spread over the device and extra blocks per tile only add their fixed cost.
    const int inv_split = b->n_tiles >= 64 ? 1 : std::min(32, (2 * TARGET_SMS + std::max(b->n_tiles, 1) - 1) / std::max(b->n_tiles, 1));
    if (inv_split > 1 && !b->inv_res.p) {
        RAPID_CHECK(b->inv_res.reserve(cd->Rpad)); RAPID_CHECK(b->inv_h1.reserve(cd->Rpad)); RAPID_CHECK(b->inv_h2.reserve(cd->Rpad));
        RAPID_CHECK(b->inv_ticket.reserve((size_t)std::max(b->n_tiles, 1)));
        RAPID_CUDA(cudaMemsetAsync(b->inv_res.p, 0, cd->Rpad * sizeof(int32_t), s));
        RAPID_CUDA(cudaMemsetAsync(b->inv_h1.p, 0, cd->Rpad * sizeof(unsigned long long), s));
        RAPID_CUDA(cudaMemsetAsync(b->inv_h2.p, 0, cd->Rpad * sizeof(unsigned long long), s));
        RAPID_CUDA(cudaMemsetAsync(b->inv_ticket.p, 0, (size_t)std::max(b->n_tiles, 1) * sizeof(int32_t), s));
    }
    ra.inv_split = inv_split; ra.inv_res = b->inv_res.p; ra.inv_h1 = b->inv_h1.p; ra.inv_h2 = b->inv_h2.p; ra.inv_ticket = b->inv_ticket.p;
    const unsigned rblocks = (unsigned)(cd->Rpad / GEN_THREADS);
    const int cgrid = std::max(1, std::min(b->resolve_grid, std::max(32, 4 * (int)rblocks)));      // co-resident (cooperative) grids
    RAPID_CHECK(b->ra_dev.reserve(sizeof(ResolveArgs)));
    // pageable source, a few hundred bytes: the driver copies it into the command stream before returning
    RAPID_CUDA(cudaMemcpyAsync(b->ra_dev.p, &ra, sizeof(ResolveArgs), cudaMemcpyHostToDevice, s));
    const ResolveArgs* ga = (const ResolveArgs*)b->ra_dev.p;
    void* args[] = {(void*)&ga};
    if (seq) {
        // the premises of the one-pass treatment, per receiver, BEFORE anything is committed (y = 0: A1, y >= 1: A2 over slot chunks)
        const unsigned echunks = (unsigned)std::max<int64_t>(1, std::min<int64_t>(64, 32 * TARGET_SMS / std::max(1u, rblocks)));
        k_seq_check<<<dim3(rblocks, 1 + echunks), GEN_THREADS, 0, s>>>(ga);
        RAPID_KERNEL_CHECK();
        cd->last_launches += 1;
    }
    k_finalize1<<<rblocks, GEN_THREADS, 0, s>>>(ga);
    RAPID_KERNEL_CHECK();
    RAPID_CUDA(cudaLaunchCooperativeKernel((void*)k_mixed_flip, dim3((unsigned)cgrid), dim3(GEN_THREADS), args, 0, s));
    k_inval_finalize2<<<(unsigned)(std::max(b->n_tiles, 1) * inv_split), GEN_THREADS, 0, s>>>(ga);
    RAPID_KERNEL_CHECK();
    RAPID_CUDA(cudaLaunchCooperativeKernel((void*)k_marks, dim3((unsigned)cgrid), dim3(GEN_THREADS), args, 0, s));
    cd->last_launches += 5;
    RAPID_CUDA(cudaMemcpyAsync(cd->h_counts.p, cd->counts_snap.p, sizeof(BatchCounts), cudaMemcpyDeviceToHost, s));
    return RAPID_OK;
}

}  // namespace rapid
