// Internal layout of the cut-detector handle (shared by cd_core.cu and cd_bucketed.cu).
#pragma once

#include <string>
#include <type_traits>
#include <vector>

#include "common.cuh"

namespace rapid {

// ---- the logical state word per (subject slot, receiver) -----------------------------------------
// bits 0..K-1 : ring r has reported the subject  (reportsPerHost[subject].containsKey(r),
//               MultiNodeCutDetector.java:92-101)
// bit 14      : sweep handles, RAW mode: emitted by the call in flight (returned list of aggregateForProposal);
//               bucketed handles: transient marker of the invalidation pass (set and cleared inside one batch)
// bit 15      : subject was emitted in a proposal (it left `proposal` at :118-121)
// preProposal == { L <= popc < H },  proposal == { popc >= H and bit 15 clear }.
// Kernels compute on this 16-bit word; how it is stored is the business of RowRef below.  Sweep handles keep bits 14 and 15 in
// their uint16 rows; bucketed rows hold the ring bits only, and their two marks live in side planes (MarkPlane).
#define CD_BIT_CALL 0x4000u
#define CD_BIT_EMIT 0x8000u

// ---- per-receiver flag word ------------------------------------------------------------------------
#define RF_SEEN_DOWN   1u   // seenLinkDownEvents           (MultiNodeCutDetector.java:88-90)
#define RF_ANNOUNCED   2u   // announcedProposal            (MembershipService.java:318, :335)
#define RF_RULE_GE_H   4u   // announced proposal == { popc >= H } (else == { bit 15 })
#define RF_ANN_NOW     8u   // announced by the batch in flight (votes in rapid_fp_tally_cd)

// Device-resident counters of a handle.  Sweep handles: initialised by the host before every batch and read back after the
// prepare kernel.  Bucketed handles: they never leave the device inside a batch — `n_slots` persists from batch to batch, the
// per-batch fields are reset by the batch's last kernel right after it copied the whole record to a snapshot the host reads at
// its next synchronisation point (no host round trip between the kernels of a batch).
struct BatchCounts {
    int32_t n_slots;       // S after slot assignment (persists across batches)
    int32_t n_valid;       // cells that passed the filter
    int32_t n_batch_subj;  // distinct subjects with at least one valid cell in this batch
    int32_t any_down;      // some valid cell has status DOWN
    int32_t bad_ring;      // index of a cell with ring >= K, or -1 (the cell is dropped, the rest of the batch applies)
    int32_t bad_dst;       // index of a cell with dst outside [0, n + joiners), or -1 (dropped likewise)
    int32_t n_mixed;       // bucketed: receivers needing exact interval resolution
    int32_t n_inval;       // bucketed: receivers that announce only the explicit part (emit marks needed)
    int32_t S_before;      // n_slots when the batch started: slots >= S_before are "fresh" (known-zero state, never read);
                           // between batches S_before == n_slots (the prepare kernel takes the slot count from here)
    int32_t overflow;      // the batch needs more subject slots than the handle holds: NOTHING was applied
    int32_t need_slots;    // ... and this many would do
    int32_t n_times;       // PERMUTED delivery: receivers whose classification needed their own crossing moments
    int32_t mixed_iters;   // fixpoint iterations of the interval analysis
    int32_t n_pairs;       // (tile, subject) pairs on the invalidation work list
    int32_t ticket;        // "last block done" counter of the resolve kernel
    int32_t serial;        // serial of the batch this record describes
    int32_t sticky_bad_ring, sticky_bad_dst, sticky_overflow;   // latched until the host collects them (asynchronous batches)
    // ---- a sequence of batches applied in one pass (see cd_bucketed.cu "sequences")
    int32_t seq_last;      // index of the last non-empty batch of the call in flight (0 for a single batch)
    int32_t seq_down;      // 1-based index of the first batch with a valid DOWN cell, INT_MAX if none
    int32_t seq_abort;     // receivers for which the one-pass treatment is not provably exact: NOTHING was committed
    int32_t mx_first;      // interval analysis: lowest flagged receiver (the reference of the uniform-delivery shortcut), INT_MAX if none
    int32_t mx_left;       // ... flagged receivers that differ from it and take the general passes
    int32_t seq_a1, seq_a2; // ... of which: could have emitted before the last batch / an implicit report would fire inside the prefix
};

struct CD {
    const View* view = nullptr;
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, evk0 = nullptr, evk1 = nullptr;
    int K = 0, H = 0, L = 0;
    uint32_t mode = 0;
    bool raw = false, bucketed = false;
    int64_t R = 0, rbegin = 0;
    uint64_t member_epoch = 0;        // the view's member_epoch at creation: receivers are ring-0 positions of THAT view
    size_t Rpad = 0;
    int nbuf = 1;                     // 2 = double-buffered rows (bucketed handles)
    int32_t S = 0;                    // slots in use (host mirror; bucketed handles: as of the last synchronisation point)
    int32_t S_before = 0;             // S when the batch in flight started (sweep handles)
    size_t S_cap = 0;
    int64_t ntot_cap = 0;             // capacity of slot_of / first_idx (node + joiner ids)

    int hb = 0;                       // bits per receiver of a row's hi plane (bucketed handles: 2 or 8), 0: uint16 rows (sweep)
    size_t row_stride = 0;            // bytes per (slot, buffer) row
    DevBuf<uint8_t> masks;            // [S_cap][nbuf] rows of row_stride bytes (see RowRef)
    DevBuf<uint32_t> emit_marks;      // [S_cap][Rpad / 32] bucketed handles: the emit plane (see MarkPlane)
    DevBuf<uint32_t> trans_marks;     // [S_cap][Rpad / 32] ... and the transient plane
    DevBuf<uint8_t> cur;              // [S_cap] which of the nbuf rows is current
    DevBuf<int32_t> slot_of;          // [ntot_cap] id -> slot, -1 if none
    DevBuf<int32_t> first_idx;        // [ntot_cap] scratch (INT_MAX)
    DevBuf<int32_t> slot_subject;     // [ntot_cap] slot -> id
    DevBuf<int32_t> touch;            // [ntot_cap] slot -> serial of the last batch that had a valid cell for it
    int32_t batch_serial = 0;
    int prep_grid_max = 0;            // co-resident blocks of the cooperative prepare kernel

    DevBuf<int32_t> n_pre;            // [R] updatesInProgress
    DevBuf<int32_t> n_prop;           // [R] proposalCount (sweep handles)
    DevBuf<uint32_t> rflags;          // [R]
    DevBuf<uint64_t> pend_h1, pend_h2;  // [R] fingerprint of `proposal` (>=H, not emitted)   (bucketed handles)
    DevBuf<int32_t> pend_cnt;         // [R]
    DevBuf<uint64_t> out_h1, out_h2;  // [R] outputs of the last batch
    DevBuf<int64_t> batch_off;        // rapid_cd_apply_batches: batch boundaries
    DevBuf<int32_t> out_batch;        // [R] ... and the batch in which each receiver announced
    DevBuf<uint64_t> sq_h1, sq_h2;    // [R] outputs of the announcing batch while a sequence is replayed batch by batch
    DevBuf<int32_t> sq_len;
    // ---- RAPID_CD_LOG: the epoch's filtered cells, for the exact replay of ONE receiver (rapid_cd_num_proposals) -------------
    struct LogRec { int64_t c0, c1; uint32_t flags; uint64_t perm_seed; int64_t blocked_off; };
    bool log_on = false, log_complete = true;
    DevBuf<int32_t> log_slot;         // per logged cell: subject slot, -1 = filtered out
    DevBuf<uint8_t> log_ring, log_status, log_blocked;
    size_t log_cells = 0, log_blocked_bytes = 0;
    std::vector<LogRec> log_batches;
    int32_t seq_merged = 0, seq_replayed = 0;   // sequences served in one pass / replayed batch by batch (diagnostics)
    int32_t seq_refused_a1 = 0, seq_refused_a2 = 0;   // receivers that failed either premise in the last refused attempt
    DevBuf<int32_t> out_len;          // [R]
    DevBuf<uint8_t> out_ann;          // [R]

    // batch staging (device)
    DevBuf<int32_t> c_dst;  DevBuf<uint8_t> c_ring, c_status;  DevBuf<int64_t> c_cfg;
    DevBuf<uint8_t> d_blocked;  DevBuf<uint32_t> d_bitmap;
    PinnedBuf<uint8_t> h_stage;  DevBuf<uint8_t> d_stage;   // host-array path: one pinned blob, one H2D copy
    const uint8_t* cur_ring_dev = nullptr;    // ring / status arrays of the batch in flight (device)
    const uint8_t* cur_status_dev = nullptr;
    DevBuf<int32_t> cell_slot;        // [A] slot or -1
    DevBuf<int32_t> scan_tmp;         // [A]
    DevBuf<int32_t> scan_sums;        // tile totals of the prefix sums
    DevBuf<BatchCounts> counts;       // [1]
    DevBuf<BatchCounts> counts_snap;  // [1] bucketed handles: copy of `counts` taken by the last kernel of a batch
    PinnedBuf<BatchCounts> h_counts;
    cudaEvent_t ev_done = nullptr;    // recorded after the last enqueued operation (other streams wait on it)
    cudaEvent_t ev_t0 = nullptr;      // rapid_cd_timer_start
    bool pending = false;             // an asynchronous batch is in flight: its status has not been collected yet
    int32_t deferred_rc = 0;          // status of asynchronous batches collected since the last rapid_cd_sync
    std::string deferred_msg;
    int32_t est_Sb = 0;               // batch subjects of the previous batch (grid sizing hint only)
    int64_t est_A = 0;
    BatchCounts last;                 // counters of the last collected batch
    int32_t retries = 0;              // batches replayed after growing the subject capacity
    // bucketed scratch lives in cd_bucketed.cu's own struct hung off here
    void* bucketed_state = nullptr;

    int32_t last_path = 0, last_launches = 0;
    int32_t last_chunks = 0, last_prep_grid = 0;   // grid of the last batch: subject chunks of the apply kernel, k_prepare blocks
    float last_ms = 0.f, last_main_ms = 0.f;
    int64_t last_A = 0;
    // the proposal census (cd_census.cu): scratch and its two output sets, created by the first census
    struct Census* census = nullptr;
};

// ---- state rows: the only code that knows how a row stores the logical words ---------------------------------------------
// Sweep handles: one interleaved uint16_t[Rpad] row per slot (the sweep kernel reads and writes one receiver per thread in place).
// Bucketed handles: every (slot, buffer) row holds ring bits only, as two planes, each padded to whole 1024-receiver tiles, back
// to back:
//   lo plane  uint8_t[Rpad]        bits 0..7 of the word (rings 0..7)
//   hi plane  Rpad lanes of HB bits, receiver r in bits [HB * r, HB * r + HB) of the plane: bits 8.. of the word
//             HB = 2 (K <= 10): rings 8, 9                            -> 1.25 B per receiver
//             HB = 8 (K <= 14): rings 8..13                           -> 2 B per receiver
// Their marks (bits 14 and 15 of the logical word) live in the MarkPlanes below.  At HB = 2 four receivers share a byte of the hi
// plane: a lane is only ever written as part of a thread-owned group of whole bytes (the group accessors, store4, the warp-wide
// row_store1_warp) — never with a plain sub-byte store.
__host__ __device__ inline int row_hi_bits(int K) { return K <= 10 ? 2 : 8; }

template <int HB>
__device__ __forceinline__ uint32_t hi_pack(uint32_t w) {      // logical word -> hi lane
    return (w >> 8) & ((1u << HB) - 1u);
}
__device__ __forceinline__ uint32_t hi_unpack(uint32_t h) {    // hi lane -> bits 8.. of the logical word
    return h << 8;
}

struct RowRef {
    uint8_t* base;
    const uint8_t* cur;
    size_t Rpad;
    size_t stride;                    // bytes per (slot, buffer) row
    int nbuf;
    int hb;                           // 0: uint16 rows (sweep); 2 / 8: two planes (bucketed)

    // lo plane of (slot, buffer); the hi plane follows it
    __device__ __forceinline__ uint8_t* lo(int32_t slot, int buf) const { return base + ((size_t)slot * nbuf + buf) * stride; }
    __device__ __forceinline__ uint8_t* cur_lo(int32_t slot) const { return lo(slot, nbuf == 2 ? cur[slot] : 0); }
    __device__ __forceinline__ uint8_t* alt_lo(int32_t slot) const { return lo(slot, cur[slot] ^ 1); }   // the non-current row (nbuf == 2)
    __device__ __forceinline__ uint16_t* row(int32_t slot) const {     // sweep handles
        return reinterpret_cast<uint16_t*>(cur_lo(slot));
    }

    // scalar get of receiver r's word in the row whose lo plane is `l`
    __device__ __forceinline__ uint32_t get(const uint8_t* l, int64_t r) const {
        if (hb == 0) return reinterpret_cast<const uint16_t*>(l)[r];
        if (hb == 2) return l[r] | hi_unpack((l[Rpad + (r >> 2)] >> ((r & 3) * 2)) & 3u);
        return l[r] | hi_unpack(l[Rpad + r]);
    }
    __device__ __forceinline__ uint32_t get(int32_t slot, int64_t r) const { return get(cur_lo(slot), r); }

    // receivers r .. r+3 (r % 4 == 0) of a bucketed row: one 32-bit lo load, one 8- or 32-bit hi load; x = lo lanes, y = hi lanes
    // (at HB = 2 the group owns exactly one byte of the hi plane)
    __device__ __forceinline__ uint2 load4(const uint8_t* l, int64_t r) const {
        return make_uint2(*reinterpret_cast<const uint32_t*>(l + r),
                          hb == 2 ? (uint32_t)l[Rpad + (r >> 2)] : *reinterpret_cast<const uint32_t*>(l + Rpad + r));
    }
    __device__ __forceinline__ uint32_t word4(uint2 g, int j) const {   // receiver r + j of a load4 group as a logical word
        return ((g.x >> (8 * j)) & 0xFFu) | hi_unpack(hb == 2 ? (g.y >> (2 * j)) & 3u : (g.y >> (8 * j)) & 0xFFu);
    }
    __device__ __forceinline__ void store4(uint8_t* l, int64_t r, const uint32_t w[4]) const {
        uint32_t lw = 0, hw = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            lw |= (w[j] & 0xFFu) << (8 * j);
            hw |= hb == 2 ? hi_pack<2>(w[j]) << (2 * j) : hi_pack<8>(w[j]) << (8 * j);
        }
        *reinterpret_cast<uint32_t*>(l + r) = lw;
        if (hb == 2) l[Rpad + (r >> 2)] = (uint8_t)hw;
        else *reinterpret_cast<uint32_t*>(l + Rpad + r) = hw;
    }
};

// 8 consecutive receivers of a bucketed row (r % 8 == 0), as SWAR lanes: lo = 8 byte lanes, hi = 8 lanes of HB bits
template <int HB>
struct Group8 {
    using Hi = typename std::conditional<HB == 2, uint16_t, uint64_t>::type;
    uint64_t lo;
    Hi hi;
};
template <int HB>
__device__ __forceinline__ const uint8_t* group8_hi(const RowRef& rows, const uint8_t* l, int64_t r) {   // the group's hi lanes
    return l + rows.Rpad + (r * HB >> 3);
}
template <int HB>
__device__ __forceinline__ Group8<HB> group8_load(const RowRef& rows, const uint8_t* l, int64_t r) {
    Group8<HB> g;
    g.lo = *reinterpret_cast<const uint64_t*>(l + r);
    g.hi = *reinterpret_cast<const typename Group8<HB>::Hi*>(group8_hi<HB>(rows, l, r));
    return g;
}
template <int HB>
__device__ __forceinline__ void group8_store(const RowRef& rows, uint8_t* l, int64_t r, const Group8<HB>& g) {
    *reinterpret_cast<uint64_t*>(l + r) = g.lo;
    *reinterpret_cast<typename Group8<HB>::Hi*>(const_cast<uint8_t*>(group8_hi<HB>(rows, l, r))) = g.hi;
}
// lane j of a group as a logical word
template <int HB>
__device__ __forceinline__ uint32_t group8_word(const Group8<HB>& g, int j) {
    return (uint32_t)((g.lo >> (8 * j)) & 0xFFu) | hi_unpack((uint32_t)(g.hi >> (HB * j)) & ((1u << HB) - 1u));
}
// lane j |= the logical bits `w`
template <int HB>
__device__ __forceinline__ void group8_or_word(Group8<HB>& g, int j, uint32_t w) {
    g.lo |= (uint64_t)(w & 0xFFu) << (8 * j);
    using Hi = typename Group8<HB>::Hi;
    g.hi = (Hi)(g.hi | ((Hi)hi_pack<HB>(w) << (HB * j)));
}
// A logical word replicated over the lanes: x = its lo byte over 4 byte lanes, y = its hi lane over 32 bits (as the lanes repeat)
template <int HB>
__device__ __forceinline__ uint2 group8_rep(uint32_t w) {
    return make_uint2((w & 0xFFu) * 0x01010101u, hi_pack<HB>(w) * (HB == 2 ? 0x55555555u : 0x01010101u));
}
// all-ones lanes for the receivers set in `act` (bit j = receiver j of the group)
template <int HB>
__device__ __forceinline__ Group8<HB> group8_mask(uint32_t act) {
    using Hi = typename Group8<HB>::Hi;
    Group8<HB> m;
    m.lo = 0; m.hi = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if ((act >> j) & 1u) { m.lo |= 0xFFull << (8 * j); m.hi = (Hi)(m.hi | ((Hi)((1u << HB) - 1u) << (HB * j))); }
    return m;
}
// the replicated word `rep` under the mask (the lanes outside it are zero)
template <int HB>
__device__ __forceinline__ Group8<HB> group8_fill(uint2 rep, const Group8<HB>& m) {
    Group8<HB> g;
    g.lo = (((uint64_t)rep.x << 32) | rep.x) & m.lo;
    g.hi = (HB == 2 ? (typename Group8<HB>::Hi)rep.y : (typename Group8<HB>::Hi)(((uint64_t)rep.y << 32) | rep.y)) & m.hi;
    return g;
}
// the lanes under the mask take the replicated word `rep`, the others keep theirs
template <int HB>
__device__ __forceinline__ void group8_merge(Group8<HB>& g, uint2 rep, const Group8<HB>& m) {
    const Group8<HB> f = group8_fill<HB>(rep, m);
    g.lo = (g.lo & ~m.lo) | f.lo;
    g.hi = (typename Group8<HB>::Hi)((g.hi & ~m.hi) | f.hi);
}
// Do all lanes under the (non-empty) mask hold the same word?  AND over them == OR over them, per plane.  *v = the OR.
// (T holds exactly 8 lanes of B bits.)
template <int B, typename T>
__device__ __forceinline__ bool lanes_same(T x, T m, uint32_t* v) {
    static_assert(B == (int)sizeof(T), "8 lanes of B bits fill the word");
    T a = (T)(x | ~m), o = (T)(x & m);
#pragma unroll
    for (int s = 4 * B; s >= B; s >>= 1) { a &= (T)(a >> s); o |= (T)(o >> s); }
    const uint32_t lm = (1u << B) - 1u;
    *v = (uint32_t)o & lm;
    return ((uint32_t)a & lm) == *v;
}
template <int HB>
__device__ __forceinline__ bool group8_same(const Group8<HB>& g, const Group8<HB>& m, uint32_t* st) {
    uint32_t vl, vh;
    const bool sl = lanes_same<8>(g.lo, m.lo, &vl);
    const bool sh = lanes_same<HB>(g.hi, m.hi, &vh);
    *st = vl | hi_unpack(vh);
    return sl && sh;
}

// one receiver per thread, consecutive threads of a warp own consecutive receivers (r % 32 == lane): every lane of the warp
// stores its word; at HB = 2 the hi lanes of 16 receivers are gathered by shuffles and one lane stores their 32-bit word
template <int HB>
__device__ __forceinline__ void row_store1_warp(const RowRef& rows, uint8_t* l, int64_t r, uint32_t w) {
    l[r] = (uint8_t)w;
    if (HB == 8) {
        l[rows.Rpad + r] = (uint8_t)hi_pack<8>(w);
    } else {
        uint32_t h = hi_pack<2>(w) << (2 * (r & 15));
        h |= __shfl_xor_sync(0xffffffffu, h, 1);
        h |= __shfl_xor_sync(0xffffffffu, h, 2);
        h |= __shfl_xor_sync(0xffffffffu, h, 4);
        h |= __shfl_xor_sync(0xffffffffu, h, 8);
        if ((r & 15) == 0) *reinterpret_cast<uint32_t*>(l + rows.Rpad + (r >> 2)) = h;
    }
}

// ---- mark planes of bucketed handles: one bit per (slot, receiver), slot-major, Rpad bits per slot, single-buffered -----------
// The apply kernels never touch them.
//   emit plane       bit 15: the subject left in the explicit-only proposal a receiver announced through the interval analysis.
//                    Written (set or clear, every slot < S) in the batch in which that receiver announces; read only while its
//                    announced rule is the explicit one, together with ">= H" (see k_gather_proposal).
//   transient plane  bit 14: raised to >= H by the invalidation pass of the batch in flight.  All zero between batches: the
//                    batch that sets bits clears them before it ends (phase_inval_unmark).
// Neighbouring receivers share a word: bits are set with atomicOr, or written by the one warp that owns the word in the pass.
struct MarkPlane {
    uint32_t* p;
    size_t words;                     // 32-bit words per slot (Rpad / 32)
    __device__ __forceinline__ uint32_t* word(int32_t slot, int64_t r) const { return p + (size_t)slot * words + (size_t)(r >> 5); }
    __device__ __forceinline__ bool test(int32_t slot, int64_t r) const { return (*word(slot, r) >> (r & 31)) & 1u; }
};

inline RowRef rowref(const CD* cd) { return RowRef{cd->masks.p, cd->cur.p, cd->Rpad, cd->row_stride, cd->nbuf, cd->hb}; }
inline MarkPlane emit_plane(const CD* cd) { return MarkPlane{cd->bucketed ? cd->emit_marks.p : nullptr, cd->Rpad / 32}; }

// Is subject slot s in the proposal receiver r announced?  rule_ge_h: r's RF_RULE_GE_H flag.  Bucketed handles (emit.p != nullptr)
// keep bit 15 in the emit plane.  That plane is written for every slot < S when the receiver announces, and never cleared: slots
// assigned later may carry marks of an earlier configuration epoch.  A mark always comes with >= H, and a receiver that has
// announced is frozen, so its word in a slot assigned later stays zero.  Requiring both therefore lists exactly the marked
// subjects of this epoch.  (rapid_cd_get_proposal and the proposal census both list proposals by this rule.)
__device__ __forceinline__ bool in_announced_proposal(const RowRef& rows, const MarkPlane& emit, int32_t s, int64_t r, int H, uint32_t RM,
                                                      int rule_ge_h) {
    const uint32_t w = rows.get(s, r);
    const bool ge_h = __popc(w & RM) >= H;
    return rule_ge_h ? ge_h : emit.p ? (ge_h && emit.test(s, r)) : ((w & CD_BIT_EMIT) != 0);
}

struct DeliveryDev {
    uint32_t flags = 0;
    const uint8_t* blocked = nullptr;
    const uint32_t* bitmap = nullptr;
    int64_t words = 0;
    uint64_t perm_seed = 0;
    int64_t cell_base = 0;            // PERMUTED: a receiver's order key of cell i is a function of i - cell_base (the index inside its batch)
};

// ---- the batch regrouped by subject (built by cd_prepare.cu, consumed by cd_bucketed.cu) -------------------------
struct SubjDesc {                     // 64 bytes, one per subject of the batch
    int32_t slot;
    uint16_t bmask;                   // rings reported in this batch (of a sequence of batches: in its LAST batch)
    uint8_t nr;                       // number of distinct rings in bmask
    uint8_t any_down;
    uint32_t tLf, tHf;                // for a fresh subject (state == pmask): moment of the cell that makes the L-th / H-th distinct ring, 0 if none
    uint32_t seg_begin, seg_len;      // its cells (of the last batch) in the slot-sorted arrays
    uint64_t mix1, mix2;              // fp_mix1 / fp_mix2 of the subject id
    // ---- a sequence of batches in one call (rapid_cd_apply_batches on bucketed handles): everything before the last batch
    uint16_t pmask;                   // rings reported in the PREFIX (batches before the last one); 0 for a single batch
    uint8_t pdown;                    // a DOWN cell in the prefix
    uint8_t pad0_;
    uint32_t f_bLp, f_bHp;            // fresh subject: 1-based prefix batch in which it reaches L / H distinct rings, 0 if it does not
    uint32_t pseg_len;                // prefix cells: they sit right before seg_begin in the sorted arrays
    uint64_t pad1_;
};
static_assert(sizeof(SubjDesc) == 64, "SubjDesc is staged in shared memory as 64-byte records");
struct SubjWalk {                     // first-occurrence ring sequence in arrival order (uniform delivery)
    uint8_t ring[16];
    uint32_t time[16];                // 1-based cell index; in a PREFIX walk (PrepOut::pwalk): 1-based batch index
};

// Invalidation work list of a bucketed handle: the subjects that sit in the unstable band of SOME receiver and have an observer
// that is itself a subject (only those can receive implicit reports, MultiNodeCutDetector.java:147-158), plus, per subject, the
// 1024-receiver tiles in which that is the case.
constexpr int SO_STRIDE = 16;
struct WorkList {
    uint8_t* has_so;                  // [slot] some observer of the subject has a slot
    int32_t* so_tab;                  // [slot][SO_STRIDE] slots of the subject's K observers (-1: not a subject)
    uint8_t* in_tile;                 // [slot][n_tiles] some receiver of the tile left the subject inside the band
    int32_t* listed;                  // [slot] on the list
    int32_t* slots;                   // the list
    int32_t* count;
    int32_t cap, n_tiles;
};
__device__ __forceinline__ void worklist_note(const WorkList& wl, int tile, int32_t slot) {
    wl.in_tile[(size_t)slot * wl.n_tiles + tile] = 1;
    if (*(volatile int32_t*)&wl.listed[slot] == 0 && atomicExch(&wl.listed[slot], 1) == 0) {
        const int32_t at = atomicAdd(wl.count, 1);
        if (at < wl.cap) wl.slots[at] = slot;
    }
}

struct PrepOut {                      // where the prepare kernel writes the regrouped batch
    SubjDesc* desc;
    SubjWalk* walk;
    int32_t* sidx;                    // cell indices grouped by subject, ascending within a subject
    uint8_t* s_ring;
    uint8_t* s_status;
    int32_t* batch_index;             // [slot] -> index of the subject in the batch
    int32_t* seg_cnt;                 // [slot] cells of the subject in this batch (scratch, all zero between batches)
    int32_t* batch_slots;             // [batch index] -> slot
    int32_t* bins;                    // [slot][64] indices of the subject's first 64 cells of this batch (any order)
    int32_t* ovf;                     // [A] cells beyond a subject's bin
    SubjWalk* pwalk;                  // sequences of batches: first-occurrence ring sequence of the prefix, time = batch index + 1
    int32_t* cell_batch;              // sequences of batches: [A] index of the batch of every valid cell
    WorkList wl;                      // invalidation work list (bucketed handles; wl.has_so == nullptr otherwise)
};

// implemented in cd_prepare.cu: filter + slot dictionary (+ regrouping by subject when po != nullptr) in ONE cooperative launch
// batch_off_dev != nullptr: the cells are a SEQUENCE of n_batches batches (cells [batch_off[b], batch_off[b+1]) = batch b) whose
// last non-empty one is `seq_last`; the descriptors then split every subject's cells into prefix and last batch.
int32_t prepare_batch(CD* cd, int64_t cfg, int64_t A, const int32_t* dst_dev, const uint8_t* ring_dev, const uint8_t* status_dev,
                      const int64_t* cfg_dev, const PrepOut* po, const int64_t* batch_off_dev = nullptr, int32_t n_batches = 1,
                      int32_t seq_last = 0);
// implemented in cd_bucketed.cu
int32_t bucketed_prep_buffers(CD* cd, int64_t A, PrepOut* po);

// enqueue only: no host synchronisation.  seq: the cells are a sequence of batches prepared with batch offsets (one pass, checked)
int32_t bucketed_apply(CD* cd, int64_t A, const DeliveryDev& dl, bool seq = false);
void bucketed_destroy(CD* cd);
int32_t bucketed_clear(CD* cd);
int32_t bucketed_clear_sticky(CD* cd);
// Wait for everything enqueued on the handle and collect the outcome of asynchronous batches (host mirrors of the slot count,
// timings, latched errors).  Returns the latched status (and clears it) when take_status is set.
int32_t cd_wait(const CD* cd, bool take_status);
// implemented in cd_census.cu
void census_destroy(CD* cd);

// ---- grouping announced proposals (cd_census.cu): the proposal census and the wire encoder's list-carrying messages ---------
// Fingerprint sources: item i takes part iff part(i); fp(i, &h1, &h2, &len) reads its fingerprint (the fp of fp_table_claim).
struct AnnouncedFp {                  // a detector's receivers that announced in its last call with at least min_len entries
    const uint32_t* rflags;
    const uint64_t* h1;
    const uint64_t* h2;
    const int32_t* len;
    int32_t min_len;
    __device__ __forceinline__ int32_t length(int32_t i) const { return len[i]; }
    __device__ __forceinline__ bool part(int32_t i) const { return (rflags[i] & RF_ANN_NOW) && (min_len <= 0 || len[i] >= min_len); }
    __device__ __forceinline__ void operator()(int32_t i, uint64_t* a, uint64_t* b, int32_t* l) const { *a = h1[i]; *b = h2[i]; *l = len[i]; }
};
struct AnswerFp {                     // acceptors' answers with a non-empty list: per answer, or (h1 == NULL) the constant (c1, c2, clen)
    const uint64_t* h1;
    const uint64_t* h2;
    const int32_t* len;
    uint64_t c1, c2;
    int32_t clen;
    __device__ __forceinline__ int32_t length(int32_t i) const { return h1 ? len[i] : clen; }
    __device__ __forceinline__ bool part(int32_t i) const { return length(i) > 0; }
    __device__ __forceinline__ void operator()(int32_t i, uint64_t* a, uint64_t* b, int32_t* l) const {
        if (h1) { *a = h1[i]; *b = h2[i]; *l = len[i]; } else { *a = c1; *b = c2; *l = clen; }
    }
};

struct GroupScal {
    int32_t n_part, n_classes, n_entries, T;
    unsigned long long entries64;     // the representatives' lengths summed in 64 bits (the int32 scan must not wrap)
};

// A grouping's scratch and per-class outputs.  Class c is the c-th representative (the lowest item of a fingerprint) in item
// order: c_h1/c_h2/c_len its fingerprint, c_rep its representative, c_voters the items that hold it, c_off the exclusive scan of
// the lengths.  The per-item arrays slot, rep, rpos and loff are free for the caller's use once group_proposals returns.
struct ProposalGroups {
    DevBuf<int32_t> table, tcnt;                                      // [T cap] open-addressing table: lowest item, voters
    DevBuf<int32_t> slot, rep, rpos, loff, scan_sums;                 // [n]
    DevBuf<uint64_t> c_h1, c_h2;                                      // [n_classes]
    DevBuf<int32_t> c_rep, c_len, c_voters, c_off, c_fill;
    DevBuf<GroupScal> sc;
    PinnedBuf<GroupScal> h_sc;                                        // the counts, on the host once group_proposals returns
    struct ListScratch* ls = nullptr;                                 // list_proposals' entry and sort scratch
    ProposalGroups() = default;
    ~ProposalGroups();
};

// Groups items [0, n) by fingerprint on stream s: cls[i] = class of item i (-1: it does not take part), and the per-class
// outputs.  One host synchronisation, before the per-class outputs are written (they are sized by the class count).
template <typename Src>
int32_t group_proposals(cudaStream_t s, int64_t n, const Src& src, ProposalGroups& g, int32_t* cls);
// The list of every class of a grouping of cd's receivers, by rapid_cd_get_proposal's rule and in its order: class c's entries
// at ids[c_off[c] ..], the status of each (DOWN: a member, UP: a registered joiner) to `status` unless it is NULL.  c_fill[c]
// counts the subjects the rule found; a class never takes more than c_len[c] of them.
int32_t list_proposals(cudaStream_t s, const CD* cd, ProposalGroups& g, int32_t* ids, uint8_t* status);

}  // namespace rapid

struct rapid_cd : rapid::CD {};
