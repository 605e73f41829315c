// Cut detector: handle lifecycle, the exact per-cell sweep kernel, accessors and the C ABI.  (Batch preparation — filter,
// subject-slot dictionary, regrouping — is cd_prepare.cu; the subject-bucketed kernels are cd_bucketed.cu.)
//
// Reference semantics (rapid/src/main/java/com/vrg/rapid/):
//   MultiNodeCutDetector.java:84-128  aggregateForProposal (per cell, in arrival order)
//   MultiNodeCutDetector.java:137-164 invalidateFailingEdges
//   MembershipService.java:300-354    batch driver (union of emissions, announcedProposal gating)
//   MembershipService.java:644-675    filterAlertMessages
// The Java keeps Map<Endpoint, Map<Integer, Endpoint>> per process; here the state of R virtual nodes is a
// [subject slot][receiver] array of ring masks in HBM (RowRef: 16-bit words, or packed planes on bucketed handles) and every
// receiver is one CUDA thread (sweep kernel) or a SWAR lane of the subject-bucketed kernels (cd_bucketed.cu).
#include <algorithm>
#include <climits>
#include <cstdlib>

#include "cd_internal.cuh"
#include "radix.cuh"

namespace rapid {

// =====================================================================================================
// preprocessing kernels
// =====================================================================================================
__global__ void k_fill_i32(int32_t* p, int64_t n, int32_t v) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// =====================================================================================================
// the sweep kernel: one thread == one receiver == one MultiNodeCutDetector, cells in arrival order
// =====================================================================================================
struct SweepArgs {
    int K, H, L, raw, do_cells, do_inval;
    int64_t R;
    RowRef rows;
    int32_t S;
    const int32_t* slot_subject;
    const int32_t* slot_of;
    const int32_t* obs;          // [id][K]: members -> ring successors, joiners -> expected observers
    int64_t A;
    const int32_t* cell_slot;
    const uint8_t* ring;
    const uint8_t* status;
    DeliveryDev dl;
    int32_t* n_pre;
    int32_t* n_prop;
    uint32_t* rflags;
    uint64_t* out_h1;
    uint64_t* out_h2;
    int32_t* out_len;
    uint8_t* out_ann;
    const int64_t* batch_off;    // NULL: the cells are ONE BatchedAlertMessage; else batch b = cells [batch_off[b], batch_off[b+1])
    int32_t n_batches;
    int32_t* out_batch;          // with batch_off: index of the batch in which the receiver announced during this call, -1 otherwise
    int64_t rbegin;              // SHUF: receiver r is global receiver rbegin + r (the key of its batch order)
};

// SHUF = false: every receiver meets the batches in array order.  SHUF = true (RAPID_DELIVERY_SHUFFLED_BATCHES): receiver r meets
// them in the order batch_order_at(batch_order_init(perm_seed, rbegin + r, n_batches), j), j = 0, 1, ...
template <bool SHUF>
__global__ void __launch_bounds__(128) k_sweep(const SweepArgs a) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.R) return;
    uint32_t flags = a.rflags[r];
    flags &= ~RF_ANN_NOW;
    if ((!a.raw && (flags & RF_ANNOUNCED)) ||                         // MembershipService.java:318-319
        ((a.dl.flags & RAPID_DELIVERY_BLOCKED) && a.dl.blocked[r])) {  // nothing delivered to this receiver
        a.rflags[r] = flags;
        a.out_h1[r] = 0; a.out_h2[r] = 0; a.out_len[r] = 0;
        if (a.out_ann) a.out_ann[r] = (flags & RF_ANNOUNCED) ? 1 : 0;
        if (a.out_batch) a.out_batch[r] = -1;
        return;
    }
    const uint32_t RM = (1u << a.K) - 1u;
    int32_t npre = a.n_pre[r], nprop = a.n_prop[r];
    bool seen = flags & RF_SEEN_DOWN;
    uint64_t oh1 = 0, oh2 = 0;
    int32_t olen = 0;
    // SHUF: whether an invalidation pass could add a report (see the rule at the pass); set at the start of the call
    bool dirty = true;

    // proposal emission (:110-121): everything at >= H that has not been emitted yet leaves in one proposal
    auto emit = [&]() {
        for (int32_t s = 0; s < a.S; ++s) {
            uint16_t* p = a.rows.row(s) + r;
            const uint32_t w = *p;
            if (!(w & CD_BIT_EMIT) && __popc(w & RM) >= a.H) {
                *p = (uint16_t)(w | CD_BIT_EMIT | (a.raw ? CD_BIT_CALL : 0u));
                const int32_t id = a.slot_subject[s];
                oh1 += fp_mix1(id);
                oh2 += fp_mix2(id);
                ++olen;
            }
        }
        ++nprop;
    };
    // one (dst slot, ring) report (:84-128); returns after updating counters
    auto report = [&](int32_t slot, int k) {
        uint16_t* p = a.rows.row(slot) + r;
        uint32_t w = *p;
        const uint32_t bit = 1u << k;
        if (w & bit) return;                               // duplicate announcement, ignore (:97-99)
        w |= bit;
        *p = (uint16_t)w;
        const int c = __popc(w & RM);
        if (c == a.L) {                                    // :104-107
            ++npre;
            if (SHUF) dirty = true;
        }
        if (c == a.H) {                                    // :109-121
            --npre;
            if (npre == 0) emit();
        }
    };

    // MembershipService.handleMessage(BatchedAlertMessage) (:300-354) once per batch, in order: the batch's cells, then
    // invalidateFailingEdges, then — if anything was emitted — announce and ignore every later batch (:318-319, :333-335)
    const bool has_bitmap = a.dl.flags & RAPID_DELIVERY_BITMAP;
    const int32_t nb = a.batch_off ? a.n_batches : 1;
    int32_t ann_batch = -1;
    BatchOrder order;
    if (SHUF) order = batch_order_init(a.dl.perm_seed, a.rbegin + r, nb);
    for (int32_t j = 0; j < nb; ++j) {
        const int32_t b = SHUF ? (int32_t)batch_order_at(order, j) : j;
        const int64_t i0 = a.batch_off ? a.batch_off[b] : 0, i1 = a.batch_off ? a.batch_off[b + 1] : a.A;
        if (a.do_cells) {
            for (int64_t i = i0; i < i1; ++i) {
                const int32_t slot = a.cell_slot[i];
                if (slot < 0) continue;
                if (has_bitmap && !((a.dl.bitmap[(size_t)i * a.dl.words + (r >> 5)] >> (r & 31)) & 1u)) continue;
                if (a.status[i] == RAPID_EDGE_DOWN) {              // :88-90 (before the duplicate check)
                    if (SHUF && !seen) dirty = true;
                    seen = true;
                }
                report(slot, a.ring[i]);
            }
        }
        // Pass skipping (SHUF, where a receiver may run a pass after each of thousands of batches).  Before an emission, in service
        // mode, U = preProposal u proposal only grows, and a pass adds implicit reports only for (n in preProposal, k) with
        // obs_k(n) in U.  A pass adds no subject to U (its reports are about subjects already at >= L) and leaves every such pair
        // reported, so the next pass can add something only if, since this one, a subject crossed L (entered U and preProposal) or
        // seenLinkDownEvents became true.  dirty records exactly that, so a skipped pass is one that would have changed nothing,
        // and the passes per receiver are bounded by #subjects + 1 instead of #batches.
        if (a.do_inval && seen && npre > 0 && (!SHUF || dirty)) {   // :137-164
            if (SHUF) dirty = false;
            for (int32_t s = 0; s < a.S; ++s) {
                const uint32_t w0 = a.rows.row(s)[r];
                const int c0 = __popc(w0 & RM);
                if (c0 < a.L || c0 >= a.H) continue;           // not in the preProposal snapshot
                const int32_t subject = a.slot_subject[s];
                for (int k = 0; k < a.K; ++k) {
                    const int32_t o = a.obs[(size_t)subject * a.K + k];
                    if (o < 0) continue;
                    const int32_t so = a.slot_of[o];
                    if (so < 0) continue;
                    const uint32_t wo = a.rows.row(so)[r];
                    if ((wo & CD_BIT_EMIT) || __popc(wo & RM) < a.L) continue;   // observer not in proposal U preProposal
                    report(s, k);                               // implicit edge report
                }
            }
        }
        if (!a.raw && olen > 0) { ann_batch = b; break; }
    }
    if (a.out_batch) a.out_batch[r] = ann_batch;
    if (seen) flags |= RF_SEEN_DOWN;
    if (!a.raw && olen > 0) flags |= RF_ANNOUNCED | RF_ANN_NOW;      // MembershipService.java:333-335
    a.rflags[r] = flags;
    a.n_pre[r] = npre;
    a.n_prop[r] = nprop;
    a.out_h1[r] = oh1;
    a.out_h2[r] = oh2;
    a.out_len[r] = olen;
    if (a.out_ann) a.out_ann[r] = (flags & RF_ANNOUNCED) ? 1 : 0;
}

// RAW mode: collect and clear the "emitted by this call" marks of one receiver
__global__ void k_gather_call(RowRef rows, int32_t S, int64_t r, const int32_t* __restrict__ slot_subject,
                              int32_t* __restrict__ out, int32_t cap, int32_t* __restrict__ count) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    uint16_t* p = rows.row(s) + r;
    const uint32_t w = *p;
    if (w & CD_BIT_CALL) {
        *p = (uint16_t)(w & ~CD_BIT_CALL);
        const int32_t at = atomicAdd(count, 1);
        if (at < cap) out[at] = slot_subject[s];
    }
}
__global__ void k_clear_call(RowRef rows, int32_t S, int64_t R) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int32_t s = blockIdx.y;
    if (r >= R || s >= S) return;
    uint16_t* p = rows.row(s) + r;
    const uint32_t w = *p;
    if (w & CD_BIT_CALL) *p = (uint16_t)(w & ~CD_BIT_CALL);
}

// the announced proposal of one receiver: (id, ring-0 key) pairs (in_announced_proposal, cd_internal.cuh)
__global__ void k_gather_proposal(RowRef rows, MarkPlane emit, int32_t S, int64_t r, int H, uint32_t RM, int rule_ge_h,
                                  const int32_t* __restrict__ slot_subject, const int64_t* __restrict__ key0,
                                  int32_t* __restrict__ out_ids, int64_t* __restrict__ out_keys, int32_t cap,
                                  int32_t* __restrict__ count) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    if (in_announced_proposal(rows, emit, s, r, H, RM, rule_ge_h)) {
        const int32_t at = atomicAdd(count, 1);
        if (at < cap) { const int32_t id = slot_subject[s]; out_ids[at] = id; out_keys[at] = key0[id]; }
    }
}

__global__ void k_dump_masks(RowRef rows, int32_t S, int64_t r, uint32_t RM, const int32_t* __restrict__ slot_subject,
                             int32_t* __restrict__ out_ids, uint16_t* __restrict__ out_masks) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    out_ids[s] = slot_subject[s];
    out_masks[s] = (uint16_t)(rows.get(s, r) & RM);
}

// S < 0: the slot count lives on the device (bucketed handles), the grid covers the handle's capacity
__global__ void k_reset_slots(int32_t S, const BatchCounts* __restrict__ bc, const int32_t* __restrict__ slot_subject,
                              int32_t* __restrict__ slot_of, uint8_t* __restrict__ cur) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (S < 0) S = bc->n_slots;
    if (s < S) { slot_of[slot_subject[s]] = -1; cur[s] = 0; }
}

// clear() of every receiver's detector scalars in one launch (MultiNodeCutDetector.java:169-178 + announcedProposal = false)
__global__ void k_clear_receivers(int64_t R, int32_t* __restrict__ n_pre, int32_t* __restrict__ n_prop, uint32_t* __restrict__ rflags,
                                  uint64_t* __restrict__ pend_h1, uint64_t* __restrict__ pend_h2, int32_t* __restrict__ pend_cnt,
                                  uint64_t* __restrict__ out_h1, uint64_t* __restrict__ out_h2, int32_t* __restrict__ out_len,
                                  uint8_t* __restrict__ out_ann) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    n_pre[r] = 0; n_prop[r] = 0; rflags[r] = 0u;
    pend_h1[r] = 0; pend_h2[r] = 0; pend_cnt[r] = 0;
    out_h1[r] = 0; out_h2[r] = 0; out_len[r] = 0; out_ann[r] = 0;
}

// =====================================================================================================
// host side
// =====================================================================================================
static int32_t ensure_id_capacity(CD* cd) {
    const int64_t ntot = cd->view->n + cd->view->nj;
    if (ntot <= cd->ntot_cap) return RAPID_OK;
    int64_t ncap = std::max<int64_t>(cd->ntot_cap, 64);
    while (ncap < ntot) ncap *= 2;
    const int64_t old = cd->ntot_cap;
    RAPID_CHECK(cd->slot_of.reserve((size_t)ncap, true, cd->stream));
    RAPID_CHECK(cd->first_idx.reserve((size_t)ncap, true, cd->stream));
    RAPID_CHECK(cd->slot_subject.reserve((size_t)ncap, true, cd->stream));
    RAPID_CHECK(cd->touch.reserve((size_t)ncap, true, cd->stream));
    ncap = (int64_t)std::min(std::min(cd->slot_of.cap, cd->touch.cap), std::min(cd->first_idx.cap, cd->slot_subject.cap));
    const int TB = 256;
    k_fill_i32<<<(unsigned)ceil_div<int64_t>(ncap - old, TB), TB, 0, cd->stream>>>(cd->slot_of.p + old, ncap - old, -1);
    k_fill_i32<<<(unsigned)ceil_div<int64_t>(ncap - old, TB), TB, 0, cd->stream>>>(cd->first_idx.p + old, ncap - old, INT_MAX);
    k_fill_i32<<<(unsigned)ceil_div<int64_t>(ncap - old, TB), TB, 0, cd->stream>>>(cd->touch.p + old, ncap - old, 0);
    RAPID_KERNEL_CHECK();
    cd->ntot_cap = ncap;
    return RAPID_OK;
}

static int32_t ensure_slot_capacity(CD* cd, size_t need) {
    if (need <= cd->S_cap) return RAPID_OK;
    size_t ncap = need;                       // first allocation: exactly what was asked for (max_subjects)
    if (cd->S_cap) { ncap = cd->S_cap; while (ncap < need) ncap *= 2; }
    const size_t row = cd->row_stride * (size_t)cd->nbuf;   // bytes per slot (both planes of every buffer of a bucketed handle)
    const size_t old_bytes = cd->S_cap * row;
    // DevBuf::reserve(keep) rounds to a power of two of elements; force the exact size instead
    DevBuf<uint8_t> nm;
    RAPID_CHECK(nm.reserve(ncap * row));
    if (old_bytes) RAPID_CUDA(cudaMemcpyAsync(nm.p, cd->masks.p, old_bytes, cudaMemcpyDeviceToDevice, cd->stream));
    RAPID_CUDA(cudaMemsetAsync(nm.p + old_bytes, 0, ncap * row - old_bytes, cd->stream));
    DevBuf<uint8_t> nc;
    RAPID_CHECK(nc.reserve(ncap));
    RAPID_CUDA(cudaMemsetAsync(nc.p, 0, ncap, cd->stream));
    if (cd->S_cap) RAPID_CUDA(cudaMemcpyAsync(nc.p, cd->cur.p, cd->S_cap, cudaMemcpyDeviceToDevice, cd->stream));
    // bucketed handles: the two mark planes grow with the rows (zero-filled: the transient plane's invariant)
    const size_t words = cd->Rpad / 32, old_words = cd->S_cap * words;
    auto grow_plane = [&](const DevBuf<uint32_t>& from, DevBuf<uint32_t>& to) -> int32_t {
        RAPID_CHECK(to.reserve(ncap * words));
        if (old_words) RAPID_CUDA(cudaMemcpyAsync(to.p, from.p, old_words * sizeof(uint32_t), cudaMemcpyDeviceToDevice, cd->stream));
        RAPID_CUDA(cudaMemsetAsync(to.p + old_words, 0, (ncap * words - old_words) * sizeof(uint32_t), cd->stream));
        return RAPID_OK;
    };
    DevBuf<uint32_t> ne, nt;
    if (cd->bucketed) {
        RAPID_CHECK(grow_plane(cd->emit_marks, ne));
        RAPID_CHECK(grow_plane(cd->trans_marks, nt));
    }
    RAPID_CUDA(cudaStreamSynchronize(cd->stream));
    std::swap(cd->masks.p, nm.p); std::swap(cd->masks.cap, nm.cap);
    std::swap(cd->cur.p, nc.p); std::swap(cd->cur.cap, nc.cap);
    if (cd->bucketed) {
        std::swap(cd->emit_marks.p, ne.p); std::swap(cd->emit_marks.cap, ne.cap);
        std::swap(cd->trans_marks.p, nt.p); std::swap(cd->trans_marks.cap, nt.cap);
    }
    cd->S_cap = ncap;
    return RAPID_OK;
}

// Sweep handles: filter the batch, give every new subject a slot, write cell_slot[]; one host sync to read the counts (the sweep
// kernel's rows must exist before it runs).  Cells with a ring number >= K or an unknown edgeDst are dropped and reported
// (RAPID_EINVAL) AFTER the rest of the batch has been applied — the Java trusts ring numbers (only `assert`,
// MultiNodeCutDetector.java:87) and never loses the valid alerts of a batch.
static int32_t preprocess(CD* cd, int64_t cfg, int64_t A, const int32_t* dst_dev, const uint8_t* ring_dev,
                          const uint8_t* status_dev, const int64_t* cfg_dev, BatchCounts* out) {
    cudaStream_t s = cd->stream;
    RAPID_CHECK(ensure_id_capacity(cd));
    RAPID_CHECK(cd->cell_slot.reserve(std::max<int64_t>(A, 1)));
    BatchCounts init;
    memset(&init, 0, sizeof(init));
    init.n_slots = cd->S;
    cd->S_before = cd->S;
    init.bad_ring = -1;
    init.bad_dst = -1;
    *cd->h_counts.p = init;
    RAPID_CUDA(cudaMemcpyAsync(cd->counts.p, cd->h_counts.p, sizeof(BatchCounts), cudaMemcpyHostToDevice, s));
    if (A > 0) {
        RAPID_CHECK(prepare_batch(cd, cfg, A, dst_dev, ring_dev, status_dev, cfg_dev, nullptr));
    } else {
        ++cd->batch_serial;
    }
    RAPID_CUDA(cudaMemcpyAsync(cd->h_counts.p, cd->counts.p, sizeof(BatchCounts), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    *out = *cd->h_counts.p;
    cd->S = out->n_slots;
    RAPID_CHECK(ensure_slot_capacity(cd, (size_t)cd->S));
    return RAPID_OK;
}

static int32_t bad_cell_status(const CD* cd, const BatchCounts& c) {
    if (c.bad_ring >= 0) { set_error("cell %d: ring number >= K (%d) (dropped; the rest of the batch was applied)", c.bad_ring, cd->K); return RAPID_EINVAL; }
    if (c.bad_dst >= 0) { set_error("cell %d: edgeDst id outside [0, members + registered joiners) (dropped; the rest of the batch was applied)", c.bad_dst); return RAPID_EINVAL; }
    return RAPID_OK;
}

// ---- bucketed handles: asynchronous batches -----------------------------------------------------------------------------
// The stream is idle: read the snapshot of the device counters the last enqueued operation left in pinned memory.
static void collect(CD* cd) {
    const BatchCounts c = *cd->h_counts.p;
    cd->last = c;
    cd->S = c.n_slots;
    if (c.n_batch_subj > 0 && cd->last_A > 0) { cd->est_Sb = c.n_batch_subj; cd->est_A = cd->last_A; }
    cudaEventElapsedTime(&cd->last_ms, cd->ev0, cd->ev1);
    cudaEventElapsedTime(&cd->last_main_ms, cd->evk0, cd->evk1);
    cudaGetLastError();
    if (c.sticky_overflow || c.sticky_bad_ring || c.sticky_bad_dst) {
        if (c.sticky_overflow) {
            cd->log_complete = false;                       // a logged batch was not applied after all
            cd->deferred_rc = RAPID_ENOMEM;
            cd->deferred_msg = "a batch needed more subject slots than the handle holds and was NOT applied (asynchronous batches cannot "
                               "grow the handle: raise max_subjects, or use the synchronous entry points)";
        } else if (cd->deferred_rc == RAPID_OK) {
            cd->deferred_rc = RAPID_EINVAL;
            cd->deferred_msg = c.sticky_bad_ring ? "a cell with ring number >= K was dropped (the rest of its batch was applied)"
                                                 : "a cell with edgeDst outside [0, members + registered joiners) was dropped (the rest of its batch was applied)";
        }
        bucketed_clear_sticky(cd);
    }
    cd->pending = false;
}

int32_t cd_wait(const CD* ccd, bool take_status) {
    CD* cd = const_cast<CD*>(ccd);
    RAPID_CUDA(cudaStreamSynchronize(cd->stream));
    if (cd->pending) collect(cd);
    if (!take_status || cd->deferred_rc == RAPID_OK) return RAPID_OK;
    const int32_t rc = cd->deferred_rc;
    set_error("%s", cd->deferred_msg.c_str());
    cd->deferred_rc = RAPID_OK;
    cd->deferred_msg.clear();
    return rc;
}

// the sweep over the handle's receivers, rows and last prepared cells
static SweepArgs sweep_args(const CD* cd, int64_t A, const uint8_t* ring_dev, const uint8_t* status_dev, const DeliveryDev& dl,
                            bool do_cells, bool do_inval, const int64_t* batch_off_dev, int32_t n_batches, int32_t* out_batch_dev) {
    SweepArgs a;
    a.batch_off = batch_off_dev; a.n_batches = n_batches; a.out_batch = out_batch_dev;
    a.K = cd->K; a.H = cd->H; a.L = cd->L; a.raw = cd->raw ? 1 : 0;
    a.do_cells = do_cells; a.do_inval = do_inval;
    a.R = cd->R;
    a.rows = rowref(cd);
    a.S = cd->S;
    a.slot_subject = cd->slot_subject.p;
    a.slot_of = cd->slot_of.p;
    a.obs = cd->view->obs.p;
    a.A = A;
    a.cell_slot = cd->cell_slot.p;
    a.ring = ring_dev;
    a.status = status_dev;
    a.dl = dl;
    a.n_pre = cd->n_pre.p; a.n_prop = cd->n_prop.p; a.rflags = cd->rflags.p;
    a.out_h1 = cd->out_h1.p; a.out_h2 = cd->out_h2.p; a.out_len = cd->out_len.p; a.out_ann = cd->out_ann.p;
    a.rbegin = cd->rbegin;
    return a;
}

static int32_t launch_sweep(CD* cd, int64_t A, const uint8_t* ring_dev, const uint8_t* status_dev, const DeliveryDev& dl,
                            bool do_cells, bool do_inval, const int64_t* batch_off_dev = nullptr, int32_t n_batches = 0,
                            int32_t* out_batch_dev = nullptr) {
    const SweepArgs a = sweep_args(cd, A, ring_dev, status_dev, dl, do_cells, do_inval, batch_off_dev, n_batches, out_batch_dev);
    const int TB = 128;
    RAPID_CUDA(cudaEventRecord(cd->evk0, cd->stream));
    if (dl.flags & RAPID_DELIVERY_SHUFFLED_BATCHES) k_sweep<true><<<(unsigned)ceil_div<int64_t>(cd->R, TB), TB, 0, cd->stream>>>(a);
    else k_sweep<false><<<(unsigned)ceil_div<int64_t>(cd->R, TB), TB, 0, cd->stream>>>(a);
    RAPID_KERNEL_CHECK();
    RAPID_CUDA(cudaEventRecord(cd->evk1, cd->stream));
    cd->last_launches += 1;
    cd->last_path = 1;
    return RAPID_OK;
}

// RAPID_DELIVERY_SHUFFLED_BATCHES is checked before anything is staged or applied, so a refusal leaves the handle as it was.
// Bucketed handles refuse it: their one-pass fold of a sequence needs one last batch shared by every receiver (DESIGN §4.3.1).
static int32_t check_shuffled(const CD* cd, const rapid_delivery* d, bool sequence) {
    if (!d || !(d->flags & RAPID_DELIVERY_SHUFFLED_BATCHES)) return RAPID_OK;
    if (!sequence) { set_error("RAPID_DELIVERY_SHUFFLED_BATCHES orders the batches of a sequence: use rapid_cd_apply_batches(_dev)"); return RAPID_EINVAL; }
    if (d->flags & (RAPID_DELIVERY_PERMUTED | RAPID_DELIVERY_BITMAP)) {
        set_error("RAPID_DELIVERY_SHUFFLED_BATCHES applies each batch's cells in array order: it cannot be combined with PERMUTED or BITMAP");
        return RAPID_EINVAL;
    }
    if (cd->bucketed || cd->raw) {
        set_error("RAPID_DELIVERY_SHUFFLED_BATCHES runs on the per-cell sweep kernel: create a SERVICE handle with RAPID_CD_SWEEP");
        return RAPID_EUNSUPPORTED;
    }
    return RAPID_OK;
}

static int32_t check_delivery(int64_t A, const rapid_delivery* d) {
    if (!d || d->flags == 0) return RAPID_OK;
    if (d->flags & ~(RAPID_DELIVERY_BLOCKED | RAPID_DELIVERY_BITMAP | RAPID_DELIVERY_PERMUTED | RAPID_DELIVERY_SHUFFLED_BATCHES)) { set_error("unknown delivery flags"); return RAPID_EINVAL; }
    if ((d->flags & RAPID_DELIVERY_BLOCKED) && !d->blocked) { set_error("delivery.blocked is NULL"); return RAPID_EINVAL; }
    if ((d->flags & RAPID_DELIVERY_BITMAP) && !d->bitmap && A) { set_error("delivery.bitmap is NULL"); return RAPID_EINVAL; }
    return RAPID_OK;
}

// a delivery that passed check_delivery; `blocked` is its receiver array in device memory (host arrays travel in the staging blob)
static int32_t upload_delivery(CD* cd, int64_t A, const rapid_delivery* d, bool on_device, const uint8_t* blocked, DeliveryDev* out) {
    *out = DeliveryDev();
    if (!d || d->flags == 0) return RAPID_OK;
    out->flags = d->flags;
    out->perm_seed = d->perm_seed;
    out->words = (cd->R + 31) / 32;
    if (d->flags & RAPID_DELIVERY_BLOCKED) out->blocked = blocked;
    if (d->flags & RAPID_DELIVERY_BITMAP) {
        if (on_device) out->bitmap = d->bitmap;
        else {
            const size_t n = (size_t)A * (size_t)out->words;
            RAPID_CHECK(cd->d_bitmap.reserve(std::max<size_t>(1, n)));
            if (n) RAPID_CUDA(cudaMemcpyAsync(cd->d_bitmap.p, d->bitmap, n * sizeof(uint32_t), cudaMemcpyHostToDevice, cd->stream));
            out->bitmap = cd->d_bitmap.p;
        }
    }
    return RAPID_OK;
}

// ---- RAPID_CD_LOG: the epoch's cells, and the exact replay of one receiver ---------------------------------------------------------
constexpr size_t LOG_MAX_CELLS = (size_t)1 << 24;

// after a batch (or a whole sequence) has been prepared: keep its filtered cells (slot per cell), ring numbers, status and the
// delivery parameters; enqueued on the handle's stream (cell_slot is overwritten by the next prepare)
static int32_t log_append(CD* cd, int64_t A, const uint8_t* ring_dev, const uint8_t* status_dev, const DeliveryDev& dl, uint64_t perm_seed_base,
                          const int64_t* batch_off_host, int32_t n_batches) {
    if (!cd->log_on || !cd->log_complete) return RAPID_OK;
    if ((dl.flags & RAPID_DELIVERY_BITMAP) || cd->log_cells + (size_t)A > LOG_MAX_CELLS) { cd->log_complete = false; return RAPID_OK; }
    cudaStream_t s = cd->stream;
    const size_t c0 = cd->log_cells, n = (size_t)A;
    if (n) {
        RAPID_CHECK(cd->log_slot.reserve(c0 + n, true, s)); RAPID_CHECK(cd->log_ring.reserve(c0 + n, true, s)); RAPID_CHECK(cd->log_status.reserve(c0 + n, true, s));
        RAPID_CUDA(cudaMemcpyAsync(cd->log_slot.p + c0, cd->cell_slot.p, n * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
        RAPID_CUDA(cudaMemcpyAsync(cd->log_ring.p + c0, ring_dev, n, cudaMemcpyDeviceToDevice, s));
        RAPID_CUDA(cudaMemcpyAsync(cd->log_status.p + c0, status_dev, n, cudaMemcpyDeviceToDevice, s));
    }
    int64_t boff = -1;
    if (dl.flags & RAPID_DELIVERY_BLOCKED) {
        boff = (int64_t)cd->log_blocked_bytes;
        RAPID_CHECK(cd->log_blocked.reserve(cd->log_blocked_bytes + (size_t)cd->R, true, s));
        RAPID_CUDA(cudaMemcpyAsync(cd->log_blocked.p + boff, dl.blocked, (size_t)cd->R, cudaMemcpyDeviceToDevice, s));
        cd->log_blocked_bytes += (size_t)cd->R;
    }
    if (batch_off_host) {
        for (int32_t b = 0; b < n_batches; ++b) {
            if (batch_off_host[b] >= A) break;
            const int64_t e = std::min<int64_t>(batch_off_host[b + 1], A);
            if (e == batch_off_host[b]) continue;
            cd->log_batches.push_back(CD::LogRec{(int64_t)c0 + batch_off_host[b], (int64_t)c0 + e, dl.flags, perm_seed_base + (uint64_t)b, boff});
        }
    } else {
        cd->log_batches.push_back(CD::LogRec{(int64_t)c0, (int64_t)(c0 + n), dl.flags, perm_seed_base, boff});
    }
    cd->log_cells += n;
    return RAPID_OK;
}

__global__ void k_replay_keys(int64_t c0, int64_t c1, uint64_t rs, uint64_t* __restrict__ key, int32_t* __restrict__ idx) {
    const int64_t i = c0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= c1) return;
    key[i - c0] = splitmix64(rs ^ (uint64_t)(i - c0));
    idx[i - c0] = (int32_t)i;
}

__global__ void k_replay_gather(int64_t n, const int32_t* __restrict__ idx, const int32_t* __restrict__ slot, const uint8_t* __restrict__ ring,
                                const uint8_t* __restrict__ status, int32_t* __restrict__ out_slot, uint8_t* __restrict__ out_ring,
                                uint8_t* __restrict__ out_status) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int32_t i = idx[j];
    out_slot[j] = slot[i]; out_ring[j] = ring[i]; out_status[j] = status[i];
}

// ---- bucketed handles: one batch (or a whole sequence of batches in one pass: batch_off_dev != nullptr) -----------------------
// Three-plus launches (prepare, apply, resolve kernels) and the copy of the counter snapshot, no host round trip in between.
// The synchronous entry points wait here and replay the batch if the handle had to grow; the asynchronous one returns.
static int32_t bucketed_one(CD* cd, int64_t cfg, int64_t A, const int32_t* dst_dev, const uint8_t* ring_dev, const uint8_t* status_dev,
                            const int64_t* cfg_dev, const DeliveryDev& dl, bool async, const int64_t* batch_off_dev = nullptr,
                            int32_t n_batches = 1, int32_t seq_last = 0, bool do_log = true) {
    cd->cur_ring_dev = ring_dev;
    cd->cur_status_dev = status_dev;
    const bool seq = batch_off_dev != nullptr && seq_last > 0;
    for (int attempt = 0;; ++attempt) {
        cd->last_launches = 0;
        cd->last_A = A;
        RAPID_CUDA(cudaEventRecord(cd->ev0, cd->stream));
        RAPID_CHECK(ensure_id_capacity(cd));
        RAPID_CHECK(cd->cell_slot.reserve(std::max<int64_t>(A, 1)));
        PrepOut po;
        RAPID_CHECK(bucketed_prep_buffers(cd, A, &po));
        if (A > 0) RAPID_CHECK(prepare_batch(cd, cfg, A, dst_dev, ring_dev, status_dev, cfg_dev, &po, seq ? batch_off_dev : nullptr, n_batches, seq_last));
        else ++cd->batch_serial;
        RAPID_CHECK(bucketed_apply(cd, A, dl, seq));
        RAPID_CUDA(cudaEventRecord(cd->ev1, cd->stream));
        RAPID_CUDA(cudaEventRecord(cd->ev_done, cd->stream));
        cd->pending = true;
        if (async) {
            if (do_log) RAPID_CHECK(log_append(cd, A, ring_dev, status_dev, dl, dl.perm_seed, nullptr, 1));   // (an overflow found later voids the log)
            return RAPID_OK;
        }
        RAPID_CUDA(cudaStreamSynchronize(cd->stream));
        const int32_t carried_rc = cd->deferred_rc;            // errors of EARLIER asynchronous batches stay latched
        const std::string carried_msg = cd->deferred_msg;
        collect(cd);
        if (cd->last.overflow && attempt < 4) {
            // not an error here: grow the handle and replay (k_prepare rolled its slot assignment back, nothing was applied)
            cd->deferred_rc = carried_rc; cd->deferred_msg = carried_msg;
            RAPID_CHECK(ensure_slot_capacity(cd, (size_t)cd->last.need_slots));
            ++cd->retries;
            continue;
        }
        if (do_log && !cd->last.overflow) RAPID_CHECK(log_append(cd, A, ring_dev, status_dev, dl, dl.perm_seed, nullptr, 1));
        const int32_t rc = bad_cell_status(cd, cd->last);
        if (rc != RAPID_OK) { cd->deferred_rc = carried_rc; cd->deferred_msg = carried_msg; return rc; }
        return RAPID_OK;
    }
}

// ---- a sequence of BatchedAlertMessages on a bucketed handle --------------------------------------------------------------------
// announced_in / outputs of a sequence: a receiver that announces in batch b keeps that batch's proposal as its output even though
// later batches of a batch-by-batch replay reset the per-batch output arrays.
__global__ void k_seq_begin(int64_t R, int32_t* __restrict__ out_batch) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < R) out_batch[r] = -1;
}
__global__ void k_seq_note(int64_t R, const uint32_t* __restrict__ rflags, int32_t b, int32_t* __restrict__ out_batch,
                           const uint64_t* __restrict__ out_h1, const uint64_t* __restrict__ out_h2, const int32_t* __restrict__ out_len,
                           uint64_t* __restrict__ sq_h1, uint64_t* __restrict__ sq_h2, int32_t* __restrict__ sq_len) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R || !(rflags[r] & RF_ANN_NOW)) return;
    out_batch[r] = b; sq_h1[r] = out_h1[r]; sq_h2[r] = out_h2[r]; sq_len[r] = out_len[r];
}
__global__ void k_seq_finish(int64_t R, uint32_t* __restrict__ rflags, const int32_t* __restrict__ out_batch,
                             uint64_t* __restrict__ out_h1, uint64_t* __restrict__ out_h2, int32_t* __restrict__ out_len,
                             const uint64_t* __restrict__ sq_h1, const uint64_t* __restrict__ sq_h2, const int32_t* __restrict__ sq_len) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R || out_batch[r] < 0) return;
    rflags[r] |= RF_ANN_NOW;                     // "announced during this call": what rapid_fp_tally_cd turns into votes
    out_h1[r] = sq_h1[r]; out_h2[r] = sq_h2[r]; out_len[r] = sq_len[r];
}

// handleMessage (MembershipService.java:300-354) once per batch, in order, for every receiver.  First the whole sequence in ONE
// pass over the state (cd_bucketed.cu, "sequences of batches in ONE pass": exact whenever its two premises hold for every
// receiver, which the device checks before committing anything); if a receiver fails the check, batch by batch.
static int32_t bucketed_sequence(CD* cd, int64_t cfg, int64_t A, const int32_t* dst_dev, const uint8_t* ring_dev, const uint8_t* status_dev,
                                 const int64_t* cfg_dev, const DeliveryDev& dl, const int64_t* off, const int64_t* batch_off_dev,
                                 int32_t n_batches, int32_t* out_batch_dev) {
    (void)A;
    cudaStream_t s = cd->stream;
    const size_t R = (size_t)cd->R;
    RAPID_CHECK(cd->sq_h1.reserve(R)); RAPID_CHECK(cd->sq_h2.reserve(R)); RAPID_CHECK(cd->sq_len.reserve(R));
    const unsigned g = (unsigned)ceil_div<int64_t>(cd->R, 256);
    k_seq_begin<<<g, 256, 0, s>>>(cd->R, out_batch_dev);
    RAPID_KERNEL_CHECK();
    auto note = [&](int32_t b) -> int32_t {
        k_seq_note<<<g, 256, 0, s>>>(cd->R, cd->rflags.p, b, out_batch_dev, cd->out_h1.p, cd->out_h2.p, cd->out_len.p,
                                     cd->sq_h1.p, cd->sq_h2.p, cd->sq_len.p);
        RAPID_KERNEL_CHECK();
        return RAPID_OK;
    };
    auto finish = [&]() -> int32_t {
        k_seq_finish<<<g, 256, 0, s>>>(cd->R, cd->rflags.p, out_batch_dev, cd->out_h1.p, cd->out_h2.p, cd->out_len.p,
                                       cd->sq_h1.p, cd->sq_h2.p, cd->sq_len.p);
        RAPID_KERNEL_CHECK();
        RAPID_CUDA(cudaEventRecord(cd->ev_done, s));
        return RAPID_OK;
    };
    auto one = [&](int32_t b) -> int32_t {                       // batch b on its own
        DeliveryDev d = dl;
        d.perm_seed = dl.perm_seed + (uint64_t)b;
        if (d.bitmap) d.bitmap = dl.bitmap + (size_t)off[b] * (size_t)dl.words;
        return bucketed_one(cd, cfg, off[b + 1] - off[b], dst_dev + off[b], ring_dev + off[b], status_dev + off[b],
                            cfg_dev ? cfg_dev + off[b] : nullptr, d, false);
    };
    int32_t first = -1, last = -1;
    for (int32_t b = 0; b < n_batches; ++b)
        if (off[b + 1] > off[b]) { if (first < 0) first = b; last = b; }
    if (last < 0) {                                              // no cells at all: handleMessage still runs invalidateFailingEdges
        RAPID_CHECK(bucketed_one(cd, cfg, 0, dst_dev, ring_dev, status_dev, cfg_dev, dl, false));
        RAPID_CHECK(note(0));
        return finish();
    }
    int32_t first_rc = RAPID_OK;
    std::string first_msg;
    auto keep = [&](int32_t rc) { if (rc != RAPID_OK && first_rc == RAPID_OK) { first_rc = rc; char buf[512]; rapid_last_error(buf, sizeof(buf)); first_msg = buf; } };
    if (first == last) {                                         // (batches without cells change nothing: the invalidation pass is idempotent)
        const int32_t rc = one(last);
        if (rc != RAPID_OK && rc != RAPID_EINVAL) return rc;
        keep(rc);
        RAPID_CHECK(note(last));
        RAPID_CHECK(finish());
        if (first_rc != RAPID_OK) { set_error("%s", first_msg.c_str()); return first_rc; }
        return RAPID_OK;
    }
    const bool mergeable = !(dl.flags & RAPID_DELIVERY_BITMAP);
    if (mergeable) {
        DeliveryDev d = dl;
        d.perm_seed = dl.perm_seed + (uint64_t)last;             // the moments that matter are those of the last batch
        d.cell_base = off[last];
        const int32_t rc = bucketed_one(cd, cfg, off[last + 1], dst_dev, ring_dev, status_dev, cfg_dev, d, false, batch_off_dev, n_batches, last, false);
        if (rc != RAPID_OK && rc != RAPID_EINVAL) return rc;
        if (!cd->last.seq_abort) {
            keep(rc);
            if (!cd->last.overflow) RAPID_CHECK(log_append(cd, off[last + 1], ring_dev, status_dev, dl, dl.perm_seed, off, n_batches));
            ++cd->seq_merged;
            RAPID_CHECK(note(last));
            RAPID_CHECK(finish());
            if (first_rc != RAPID_OK) { set_error("%s", first_msg.c_str()); return first_rc; }
            return RAPID_OK;
        }
        // refused for some receiver: nothing was committed — batch by batch (bad cells are reported by the replay)
        cd->seq_refused_a1 = cd->last.seq_a1; cd->seq_refused_a2 = cd->last.seq_a2;
    }
    ++cd->seq_replayed;
    for (int32_t b = first; b <= last; ++b) {
        if (off[b + 1] == off[b]) continue;
        const int32_t rc = one(b);
        if (rc != RAPID_OK && rc != RAPID_EINVAL) return rc;
        keep(rc);
        RAPID_CHECK(note(b));
    }
    RAPID_CHECK(finish());
    if (first_rc != RAPID_OK) { set_error("%s", first_msg.c_str()); return first_rc; }
    return RAPID_OK;
}

static int32_t apply_common(CD* cd, int64_t cfg, int64_t A, const int32_t* dst_dev, const uint8_t* ring_dev,
                            const uint8_t* status_dev, const int64_t* cfg_dev, const DeliveryDev& dl,
                            const int64_t* batch_off_dev = nullptr, int32_t n_batches = 0, int32_t* out_batch_dev = nullptr,
                            bool async = false, const int64_t* batch_off_host = nullptr) {
    cd->cur_ring_dev = ring_dev;
    cd->cur_status_dev = status_dev;
    if (cd->bucketed) {
        if (batch_off_dev) return bucketed_sequence(cd, cfg, A, dst_dev, ring_dev, status_dev, cfg_dev, dl, batch_off_host, batch_off_dev, n_batches, out_batch_dev);
        return bucketed_one(cd, cfg, A, dst_dev, ring_dev, status_dev, cfg_dev, dl, async);
    }
    cd->last_launches = 0;
    cd->last_A = A;
    RAPID_CUDA(cudaEventRecord(cd->ev0, cd->stream));
    BatchCounts bc;
    RAPID_CHECK(preprocess(cd, cfg, A, dst_dev, ring_dev, status_dev, cfg_dev, &bc));
    RAPID_CHECK(launch_sweep(cd, A, ring_dev, status_dev, dl, true, !cd->raw, batch_off_dev, n_batches, out_batch_dev));
    RAPID_CUDA(cudaEventRecord(cd->ev1, cd->stream));
    RAPID_CUDA(cudaEventRecord(cd->ev_done, cd->stream));
    RAPID_CUDA(cudaStreamSynchronize(cd->stream));
    cudaEventElapsedTime(&cd->last_ms, cd->ev0, cd->ev1);
    cudaEventElapsedTime(&cd->last_main_ms, cd->evk0, cd->evk1);
    cd->last = bc;
    return bad_cell_status(cd, bc);
}

// Host arrays -> one pinned blob -> ONE host-to-device copy.  Layout: [cfg int64 x n]? [dst int32 x n] [ring u8 x n]
// [status u8 x n] [blocked u8 x R]?  (8-byte things first so every section is naturally aligned)
struct Staged { const int32_t* dst; const uint8_t* ring; const uint8_t* status; const int64_t* cfg; const uint8_t* blocked; };

static int32_t stage_cells(rapid_cd* cd, int64_t n, const int32_t* dst, const uint8_t* ring, const uint8_t* status, const int64_t* cfg,
                           const uint8_t* blocked, Staged* out) {
    const size_t un = (size_t)n, R = (size_t)cd->R;
    const size_t o_cfg = 0, o_dst = o_cfg + (cfg ? 8 * un : 0), o_ring = o_dst + 4 * un, o_status = o_ring + un;
    const size_t o_blk = (o_status + un + 7) & ~(size_t)7, total = o_blk + (blocked ? R : 0);
    RAPID_CHECK(cd->h_stage.reserve(std::max<size_t>(total, 8)));
    RAPID_CHECK(cd->d_stage.reserve(std::max<size_t>(total, 8)));
    uint8_t* h = cd->h_stage.p;
    if (cfg) memcpy(h + o_cfg, cfg, 8 * un);
    if (un) { memcpy(h + o_dst, dst, 4 * un); memcpy(h + o_ring, ring, un); memcpy(h + o_status, status, un); }
    if (blocked) memcpy(h + o_blk, blocked, R);
    if (total) RAPID_CUDA(cudaMemcpyAsync(cd->d_stage.p, h, total, cudaMemcpyHostToDevice, cd->stream));
    const uint8_t* d = cd->d_stage.p;
    out->cfg = cfg ? (const int64_t*)(d + o_cfg) : nullptr;
    out->dst = (const int32_t*)(d + o_dst);
    out->ring = d + o_ring;
    out->status = d + o_status;
    out->blocked = blocked ? d + o_blk : nullptr;
    return RAPID_OK;
}

// The one front door of the rapid_cd_apply_batch* entry points.  Every argument is checked before anything is enqueued, so a
// refused call leaves the handle exactly as it was; then host arrays are staged, the delivery and a sequence's batch offsets
// uploaded, and the batch applied.  *applied: apply_common ran (its RAPID_EINVAL means bad cells were dropped, the rest applied).
static int32_t apply_entry(rapid_cd* cd, int64_t cfg, int64_t n, const int32_t* dst, const uint8_t* ring, const uint8_t* status,
                           const int64_t* cell_cfg, const rapid_delivery* d, bool on_device, bool async, bool sequence = false,
                           int64_t n_batches = 0, const int64_t* batch_off = nullptr, bool* applied = nullptr) {
    if (!cd || n < 0 || (n && (!dst || !ring || !status)) ||
        (sequence && (n_batches < 0 || n_batches > 0x7ffffff0LL || !batch_off))) { set_error("bad arguments"); return RAPID_EINVAL; }
    RAPID_CHECK(check_delivery(n, d));
    RAPID_CHECK(check_shuffled(cd, d, sequence));
    if (async && !cd->bucketed) { set_error("asynchronous batches run on the subject-bucketed kernels (SERVICE / BUCKETED handles)"); return RAPID_EUNSUPPORTED; }
    if (cd->raw) { set_error("RAW handles take rapid_cd_aggregate / rapid_cd_invalidate"); return RAPID_EINVAL; }
    if (!cd->bucketed && d && (d->flags & RAPID_DELIVERY_PERMUTED)) { set_error("the sweep kernel applies cells in array order; RAPID_DELIVERY_PERMUTED needs a bucketed handle"); return RAPID_EUNSUPPORTED; }
    if (sequence) {
        if (batch_off[0] != 0 || batch_off[n_batches] != n) { set_error("batch_off must run from 0 to n_cells"); return RAPID_EINVAL; }
        for (int64_t b = 0; b < n_batches; ++b)
            if (batch_off[b + 1] < batch_off[b]) { set_error("batch_off must be non-decreasing"); return RAPID_EINVAL; }
    }
    DeviceGuard g(cd->device);
    const uint8_t* blocked = (d && (d->flags & RAPID_DELIVERY_BLOCKED)) ? d->blocked : nullptr;
    if (!on_device) {
        Staged st;
        RAPID_CHECK(stage_cells(cd, n, dst, ring, status, cell_cfg, blocked, &st));
        dst = st.dst; ring = st.ring; status = st.status; cell_cfg = st.cfg; blocked = st.blocked;
    }
    DeliveryDev dl;
    RAPID_CHECK(upload_delivery(cd, n, d, on_device, blocked, &dl));
    if (sequence) {
        RAPID_CHECK(cd->batch_off.reserve((size_t)n_batches + 1));
        RAPID_CHECK(cd->out_batch.reserve((size_t)cd->Rpad));
        RAPID_CUDA(cudaMemcpyAsync(cd->batch_off.p, batch_off, (size_t)(n_batches + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, cd->stream));
    }
    if (applied) *applied = true;
    return apply_common(cd, cfg, n, dst, ring, status, cell_cfg, dl, sequence ? cd->batch_off.p : nullptr, (int32_t)n_batches,
                        sequence ? cd->out_batch.p : nullptr, async, sequence ? batch_off : nullptr);
}

// getNumProposals of ONE receiver of a bucketed handle: the sweep kernel on that receiver alone, over the epoch's logged cells in
// the receiver's own order (the bucketed kernels never see a receiver's cells in order, so they cannot count emissions; the log can)
static int32_t replay_num_proposals(CD* cd, int64_t receiver, int32_t* out) {
    if (!cd->log_on) { set_error("getNumProposals on the subject-bucketed kernels replays the epoch's cell log: create the handle with RAPID_CD_LOG (or use a RAPID_CD_SWEEP handle)"); return RAPID_EUNSUPPORTED; }
    if (!cd->log_complete) { set_error("the epoch's cell log is incomplete (a per-receiver BITMAP delivery, more than 2^24 cells, or a batch that was not applied)"); return RAPID_EUNSUPPORTED; }
    cudaStream_t s = cd->stream;
    const int32_t S = cd->S;
    if (cd->log_batches.empty() || S == 0) { *out = 0; return RAPID_OK; }
    // the receiver's byte of every logged blocked array
    const size_t R = (size_t)cd->R;
    std::vector<uint8_t> blk(cd->log_blocked_bytes / R);
    if (!blk.empty()) RAPID_CUDA(cudaMemcpy2DAsync(blk.data(), 1, cd->log_blocked.p + receiver, R, 1, blk.size(), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    // the batches delivered to the receiver, their cells concatenated in log order (a blocked batch never reaches handleMessage,
    // so it has no invalidation pass either)
    std::vector<const CD::LogRec*> kept;
    std::vector<int64_t> off(1, 0);
    std::vector<int32_t> idx;
    for (const CD::LogRec& r : cd->log_batches) {
        if (r.blocked_off >= 0 && blk[(size_t)r.blocked_off / R]) continue;
        kept.push_back(&r);
        for (int64_t i = r.c0; i < r.c1; ++i) idx.push_back((int32_t)i);
        off.push_back((int64_t)idx.size());
    }
    const size_t n = idx.size(), nk = kept.size();
    struct Receiver { int32_t n_pre, n_prop, len; uint32_t rflags; uint64_t h1, h2; };
    DevBuf<int32_t> d_idx, kidx, g_slot;
    DevBuf<uint8_t> g_ring, g_status;
    DevBuf<int64_t> d_off;
    DevBuf<uint64_t> key, skey;
    DevBuf<uint16_t> rows;
    DevBuf<Receiver> one;
    RadixScratch sc;
    RAPID_CHECK(d_idx.reserve(std::max<size_t>(n, 1))); RAPID_CHECK(g_slot.reserve(std::max<size_t>(n, 1)));
    RAPID_CHECK(g_ring.reserve(std::max<size_t>(n, 1))); RAPID_CHECK(g_status.reserve(std::max<size_t>(n, 1)));
    RAPID_CHECK(d_off.reserve(nk + 1)); RAPID_CHECK(rows.reserve((size_t)S)); RAPID_CHECK(one.reserve(1));
    if (n) RAPID_CUDA(cudaMemcpyAsync(d_idx.p, idx.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    for (size_t b = 0; b < nk; ++b) {
        const CD::LogRec& r = *kept[b];
        if (!(r.flags & RAPID_DELIVERY_PERMUTED) || r.c1 == r.c0) continue;
        // this receiver's own order of the batch: ascending splitmix64(rs ^ index inside the batch)
        const int64_t nc = r.c1 - r.c0;
        RAPID_CHECK(key.reserve((size_t)nc)); RAPID_CHECK(skey.reserve((size_t)nc)); RAPID_CHECK(kidx.reserve((size_t)nc));
        k_replay_keys<<<(unsigned)ceil_div<int64_t>(nc, 256), 256, 0, s>>>(r.c0, r.c1, splitmix64(r.perm_seed + (uint64_t)(cd->rbegin + receiver)),
                                                                          key.p, kidx.p);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(radix_sort_pairs<uint64_t>(sc, key.p, kidx.p, skey.p, d_idx.p + off[b], nc, 0, 64, s));
    }
    if (n) {
        k_replay_gather<<<(unsigned)ceil_div<int64_t>((int64_t)n, 256), 256, 0, s>>>((int64_t)n, d_idx.p, cd->log_slot.p, cd->log_ring.p,
                                                                                    cd->log_status.p, g_slot.p, g_ring.p, g_status.p);
        RAPID_KERNEL_CHECK();
    }
    RAPID_CUDA(cudaMemcpyAsync(d_off.p, off.data(), (nk + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    RAPID_CUDA(cudaMemsetAsync(rows.p, 0, (size_t)S * sizeof(uint16_t), s));
    RAPID_CUDA(cudaMemsetAsync(one.p, 0, sizeof(Receiver), s));
    // the batches of one launch: the sweep stops at the batch in which the receiver announces (MembershipService.java:318-319)
    SweepArgs a = sweep_args(cd, (int64_t)n, g_ring.p, g_status.p, DeliveryDev(), true, true, d_off.p, (int32_t)nk, nullptr);
    a.R = 1;
    a.rows = RowRef{reinterpret_cast<uint8_t*>(rows.p), nullptr, 1, sizeof(uint16_t), 1, 0};
    a.cell_slot = g_slot.p;
    a.n_pre = &one.p->n_pre; a.n_prop = &one.p->n_prop; a.rflags = &one.p->rflags;
    a.out_h1 = &one.p->h1; a.out_h2 = &one.p->h2; a.out_len = &one.p->len; a.out_ann = nullptr;
    k_sweep<false><<<1, 1, 0, s>>>(a);
    RAPID_KERNEL_CHECK();
    RAPID_CUDA(cudaMemcpyAsync(out, &one.p->n_prop, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

}  // namespace rapid

using namespace rapid;

extern "C" {

int32_t rapid_cd_create(rapid_cd** out, const rapid_view* v, int32_t H, int32_t L, int64_t n_receivers,
                        int64_t receiver_begin, uint32_t mode_flags, int64_t max_subjects) {
    if (!out || !v) { set_error("NULL argument"); return RAPID_EINVAL; }
    *out = nullptr;
    const View* view = v;
    const int K = view->K;
    if (H > K || L > H || K < 3 || L <= 0 || H <= 0) {                  // MultiNodeCutDetector.java:52-55
        set_error("Arguments do not satisfy K > H >= L >= 0: (K: %d, H: %d, L: %d", K, H, L);
        return RAPID_EINVAL;
    }
    if (n_receivers < 1 || receiver_begin < 0) { set_error("bad receiver range"); return RAPID_EINVAL; }
    const bool raw = mode_flags & RAPID_CD_RAW;
    if ((mode_flags & RAPID_CD_SWEEP) && (mode_flags & RAPID_CD_BUCKETED)) { set_error("SWEEP and BUCKETED are exclusive"); return RAPID_EINVAL; }
    if (raw && (mode_flags & RAPID_CD_BUCKETED)) { set_error("RAW mode runs on the sweep kernel only"); return RAPID_EINVAL; }
    if (!raw && view->n > 0 && receiver_begin + n_receivers > view->n) { set_error("receiver range exceeds the ring"); return RAPID_EINVAL; }
    DeviceGuard g(view->device);
    rapid_cd* cd = new rapid_cd();
    cd->view = view;
    cd->member_epoch = view->member_epoch;
    cd->device = view->device;
    cd->K = K; cd->H = H; cd->L = L;
    cd->mode = mode_flags;
    cd->raw = raw;
    cd->bucketed = !raw && !(mode_flags & RAPID_CD_SWEEP);
    cd->log_on = cd->bucketed && (mode_flags & RAPID_CD_LOG);
    cd->nbuf = cd->bucketed ? 2 : 1;
    cd->R = n_receivers;
    cd->rbegin = receiver_begin;
    // rows are 256-byte multiples; bucketed handles pad to whole 1024-receiver tiles so every uint4 access is in-bounds
    const int64_t pad = cd->bucketed ? 1024 : 128;
    cd->Rpad = (size_t)ceil_div<int64_t>(n_receivers, pad) * pad;
    cd->hb = cd->bucketed ? row_hi_bits(K) : 0;
    cd->row_stride = cd->bucketed ? cd->Rpad + cd->Rpad * cd->hb / 8 : cd->Rpad * sizeof(uint16_t);
    int32_t rc = RAPID_OK;
    do {
        if (cudaStreamCreateWithFlags(&cd->stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreate(&cd->ev0) != cudaSuccess || cudaEventCreate(&cd->ev1) != cudaSuccess ||
            cudaEventCreate(&cd->evk0) != cudaSuccess || cudaEventCreate(&cd->evk1) != cudaSuccess ||
            cudaEventCreateWithFlags(&cd->ev_done, cudaEventDisableTiming) != cudaSuccess || cudaEventCreate(&cd->ev_t0) != cudaSuccess) {
            rc = cuda_fail(cudaGetLastError(), "stream/event create", __FILE__, __LINE__); break;
        }
        const size_t R = (size_t)cd->Rpad;
        if ((rc = cd->n_pre.reserve(R))) break;
        if ((rc = cd->n_prop.reserve(R))) break;
        if ((rc = cd->rflags.reserve(R))) break;
        if ((rc = cd->pend_h1.reserve(R))) break;
        if ((rc = cd->pend_h2.reserve(R))) break;
        if ((rc = cd->pend_cnt.reserve(R))) break;
        if ((rc = cd->out_h1.reserve(R))) break;
        if ((rc = cd->out_h2.reserve(R))) break;
        if ((rc = cd->out_len.reserve(R))) break;
        if ((rc = cd->out_ann.reserve(R))) break;
        if ((rc = cd->counts.reserve(1))) break;
        if ((rc = cd->counts_snap.reserve(1))) break;
        if ((rc = cd->h_counts.reserve(1))) break;
        memset(cd->h_counts.p, 0, sizeof(BatchCounts));
        // the device counters must be valid BEFORE the first clear(): it resets "the slots in use" and reads their number
        if (cudaMemsetAsync(cd->counts.p, 0, sizeof(BatchCounts), cd->stream) != cudaSuccess ||
            cudaMemsetAsync(cd->counts_snap.p, 0, sizeof(BatchCounts), cd->stream) != cudaSuccess) {
            rc = cuda_fail(cudaGetLastError(), "memset", __FILE__, __LINE__); break;
        }
        memset(&cd->last, 0, sizeof(BatchCounts));
        if ((rc = ensure_id_capacity(cd))) break;
        if ((rc = ensure_slot_capacity(cd, (size_t)std::max<int64_t>(max_subjects, 16)))) break;
        rc = rapid_cd_clear(cd);
    } while (0);
    if (rc) { rapid_cd_destroy(cd); return rc; }
    *out = cd;
    return RAPID_OK;
}

int32_t rapid_cd_destroy(rapid_cd* cd) {
    if (!cd) return RAPID_OK;
    DeviceGuard g(cd->device);
    if (cd->stream) cudaStreamSynchronize(cd->stream);
    bucketed_destroy(cd);
    census_destroy(cd);
    if (cd->ev0) cudaEventDestroy(cd->ev0);
    if (cd->ev1) cudaEventDestroy(cd->ev1);
    if (cd->evk0) cudaEventDestroy(cd->evk0);
    if (cd->evk1) cudaEventDestroy(cd->evk1);
    if (cd->ev_done) cudaEventDestroy(cd->ev_done);
    if (cd->ev_t0) cudaEventDestroy(cd->ev_t0);
    if (cd->stream) cudaStreamDestroy(cd->stream);
    delete cd;
    return RAPID_OK;
}

int32_t rapid_cd_clear(rapid_cd* cd) {
    if (!cd) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    cudaStream_t s = cd->stream;
    const size_t R = cd->Rpad;
    if (cd->bucketed) {
        // Bucketed handles never read the state of a slot before the batch that assigns it has written it (slots >= S_before
        // are write-only), so clear() is O(#slots + #receivers): forget the dictionary, reset the receivers' scalars, the work
        // list and the device counters — ONE launch, no host round trip (the slot count lives on the device).
        // The mark planes need nothing either: the transient plane is all zero between batches, and the emit plane is only read
        // for a receiver that announced in the new epoch, whose mark pass rewrites every slot it had, together with ">= H"
        // (k_gather_proposal), which the zero words of slots assigned after that never meet.
        cd->S = 0;
        RAPID_CHECK(bucketed_clear(cd));
        cd->log_cells = 0; cd->log_blocked_bytes = 0; cd->log_batches.clear(); cd->log_complete = true;
    } else {
        if (cd->S > 0) {
            k_reset_slots<<<(unsigned)ceil_div<int32_t>(cd->S, 256), 256, 0, s>>>(cd->S, cd->counts.p, cd->slot_subject.p, cd->slot_of.p, cd->cur.p);
            RAPID_KERNEL_CHECK();
            // the sweep kernel reads in place and needs zeros
            RAPID_CUDA(cudaMemsetAsync(cd->masks.p, 0, (size_t)cd->S * cd->nbuf * cd->row_stride, s));
        }
        cd->S = 0;
        k_clear_receivers<<<(unsigned)ceil_div<size_t>(R, 256), 256, 0, s>>>((int64_t)R, cd->n_pre.p, cd->n_prop.p, cd->rflags.p, cd->pend_h1.p,
                                                                            cd->pend_h2.p, cd->pend_cnt.p, cd->out_h1.p, cd->out_h2.p,
                                                                            cd->out_len.p, cd->out_ann.p);
        RAPID_KERNEL_CHECK();
    }
    if (cd->bucketed) {
        RAPID_CUDA(cudaMemcpyAsync(cd->h_counts.p, cd->counts_snap.p, sizeof(BatchCounts), cudaMemcpyDeviceToHost, s));
        cd->last_A = 0;
        cd->pending = true;
    }
    RAPID_CUDA(cudaEventRecord(cd->ev_done, s));
    // no synchronisation: everything that follows runs on the same stream, and other streams (the tally) wait on ev_done
    return RAPID_OK;
}

int32_t rapid_cd_timer_start(rapid_cd* cd) {
    if (!cd) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    RAPID_CUDA(cudaEventRecord(cd->ev_t0, cd->stream));
    RAPID_CUDA(cudaEventRecord(cd->ev_done, cd->stream));
    return RAPID_OK;
}

int32_t rapid_cd_sync(rapid_cd* cd) {
    if (!cd) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    return cd_wait(cd, true);
}

int32_t rapid_cd_read_outputs(const rapid_cd* cd, uint64_t* h1, uint64_t* h2, int32_t* len, uint8_t* ann) {
    if (!cd) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    RAPID_CHECK(cd_wait(cd, false));     // clear() and asynchronous batches are still in flight on the handle's stream
    const size_t R = (size_t)cd->R;
    if (h1) RAPID_CUDA(cudaMemcpyAsync(h1, cd->out_h1.p, R * sizeof(uint64_t), cudaMemcpyDeviceToHost, cd->stream));
    if (h2) RAPID_CUDA(cudaMemcpyAsync(h2, cd->out_h2.p, R * sizeof(uint64_t), cudaMemcpyDeviceToHost, cd->stream));
    if (len) RAPID_CUDA(cudaMemcpyAsync(len, cd->out_len.p, R * sizeof(int32_t), cudaMemcpyDeviceToHost, cd->stream));
    if (ann) RAPID_CUDA(cudaMemcpyAsync(ann, cd->out_ann.p, R, cudaMemcpyDeviceToHost, cd->stream));
    RAPID_CUDA(cudaStreamSynchronize(cd->stream));
    return RAPID_OK;
}

int32_t rapid_cd_apply_batch_dev(rapid_cd* cd, int64_t cfg_id, int64_t n_cells, const int32_t* src_dev, const int32_t* dst_dev,
                                 const uint8_t* ring_dev, const uint8_t* status_dev, const int64_t* cell_cfg_dev,
                                 const rapid_delivery* delivery_dev) {
    (void)src_dev;   // edgeSrc is stored by the Java but never read back (MultiNodeCutDetector.java:101)
    return apply_entry(cd, cfg_id, n_cells, dst_dev, ring_dev, status_dev, cell_cfg_dev, delivery_dev, /*on_device=*/true, /*async=*/false);
}

int32_t rapid_cd_apply_batch_dev_async(rapid_cd* cd, int64_t cfg_id, int64_t n_cells, const int32_t* src_dev, const int32_t* dst_dev,
                                       const uint8_t* ring_dev, const uint8_t* status_dev, const int64_t* cell_cfg_dev,
                                       const rapid_delivery* delivery_dev) {
    (void)src_dev;
    return apply_entry(cd, cfg_id, n_cells, dst_dev, ring_dev, status_dev, cell_cfg_dev, delivery_dev, /*on_device=*/true, /*async=*/true);
}

int32_t rapid_cd_apply_batch(rapid_cd* cd, int64_t cfg_id, int64_t n_cells, const int32_t* src, const int32_t* dst,
                             const uint8_t* ring, const uint8_t* status, const int64_t* cell_cfg,
                             const rapid_delivery* delivery, uint64_t* proposal_hash, uint64_t* proposal_hash2,
                             int32_t* proposal_len, uint8_t* announced) {
    (void)src;
    RAPID_CHECK(apply_entry(cd, cfg_id, n_cells, dst, ring, status, cell_cfg, delivery, /*on_device=*/false, /*async=*/false));
    if (proposal_hash || proposal_hash2 || proposal_len || announced)
        return rapid_cd_read_outputs(cd, proposal_hash, proposal_hash2, proposal_len, announced);
    return RAPID_OK;
}

// A sequence of BatchedAlertMessages — one per sender, as AlertBatcher (MembershipService.java:613-637) produces them —
// delivered to every receiver in array order, with handleMessage's gating between them.
int32_t rapid_cd_apply_batches(rapid_cd* cd, int64_t cfg_id, int64_t n_cells, const int32_t* src, const int32_t* dst, const uint8_t* ring,
                               const uint8_t* status, const int64_t* cell_cfg, int64_t n_batches, const int64_t* batch_off,
                               const rapid_delivery* delivery, uint64_t* proposal_hash, uint64_t* proposal_hash2, int32_t* proposal_len,
                               uint8_t* announced, int32_t* announced_in) {
    (void)src;
    bool applied = false;
    const int32_t rc = apply_entry(cd, cfg_id, n_cells, dst, ring, status, cell_cfg, delivery, /*on_device=*/false, /*async=*/false,
                                   /*sequence=*/true, n_batches, batch_off, &applied);
    if (!applied || (rc != RAPID_OK && rc != RAPID_EINVAL)) return rc;   // RAPID_EINVAL: bad cells were dropped, the rest was applied
    DeviceGuard g(cd->device);
    char msg[512];
    if (rc != RAPID_OK) rapid_last_error(msg, sizeof(msg));
    RAPID_CHECK(cd_wait(cd, false));
    if (announced_in) RAPID_CUDA(cudaMemcpy(announced_in, cd->out_batch.p, (size_t)cd->R * sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (proposal_hash || proposal_hash2 || proposal_len || announced)
        RAPID_CHECK(rapid_cd_read_outputs(cd, proposal_hash, proposal_hash2, proposal_len, announced));
    if (rc != RAPID_OK) set_error("%s", msg);
    return rc;
}

// The same with the cell arrays already in device memory (batch_off stays a HOST array: the host walks the batches when the
// one-pass treatment is refused).  Outputs: rapid_cd_read_outputs / rapid_cd_read_announced_in, or straight into rapid_fp_tally_cd.
int32_t rapid_cd_apply_batches_dev(rapid_cd* cd, int64_t cfg_id, int64_t n_cells, const int32_t* src_dev, const int32_t* dst_dev,
                                   const uint8_t* ring_dev, const uint8_t* status_dev, const int64_t* cell_cfg_dev, int64_t n_batches,
                                   const int64_t* batch_off, const rapid_delivery* delivery_dev) {
    (void)src_dev;
    return apply_entry(cd, cfg_id, n_cells, dst_dev, ring_dev, status_dev, cell_cfg_dev, delivery_dev, /*on_device=*/true, /*async=*/false,
                       /*sequence=*/true, n_batches, batch_off);
}

int32_t rapid_cd_read_announced_in(const rapid_cd* cd, int32_t* announced_in) {
    if (!cd || !announced_in) { set_error("NULL argument"); return RAPID_EINVAL; }
    if (!cd->out_batch.p) { set_error("no rapid_cd_apply_batches call yet"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    RAPID_CHECK(cd_wait(cd, false));
    RAPID_CUDA(cudaMemcpy(announced_in, cd->out_batch.p, (size_t)cd->R * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return RAPID_OK;
}

// diagnostics: sequences served in one pass / replayed batch by batch since the handle was created
int32_t rapid_cd_sequence_stats(const rapid_cd* cd, int32_t* one_pass, int32_t* replayed, int32_t* refused_a1, int32_t* refused_a2) {
    if (!cd) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (one_pass) *one_pass = cd->seq_merged;
    if (replayed) *replayed = cd->seq_replayed;
    if (refused_a1) *refused_a1 = cd->seq_refused_a1;
    if (refused_a2) *refused_a2 = cd->seq_refused_a2;
    return RAPID_OK;
}

// RAW mode, after a sweep: what the call emitted for `receiver` (ascending; at most cap ids, *out_len = all of them), then the
// call marks of every receiver cleared
static int32_t take_call_marks(rapid_cd* cd, int64_t receiver, int32_t* out_ids, int32_t cap, int32_t* out_len) {
    DevBuf<int32_t> d_ids, d_cnt;
    const int32_t S = cd->S;
    RAPID_CHECK(d_ids.reserve((size_t)std::max(S, 1)));
    RAPID_CHECK(d_cnt.reserve(1));
    RAPID_CUDA(cudaMemsetAsync(d_cnt.p, 0, sizeof(int32_t), cd->stream));
    int32_t n = 0;
    if (S > 0) {
        k_gather_call<<<(unsigned)ceil_div<int32_t>(S, 256), 256, 0, cd->stream>>>(rowref(cd), S, receiver, cd->slot_subject.p, d_ids.p, S, d_cnt.p);
        dim3 grid((unsigned)ceil_div<int64_t>(cd->R, 256), (unsigned)S);
        k_clear_call<<<grid, 256, 0, cd->stream>>>(rowref(cd), S, cd->R);
        RAPID_KERNEL_CHECK();
        RAPID_CUDA(cudaMemcpyAsync(&n, d_cnt.p, sizeof(int32_t), cudaMemcpyDeviceToHost, cd->stream));
    }
    RAPID_CUDA(cudaStreamSynchronize(cd->stream));
    std::vector<int32_t> ids((size_t)n);
    if (n) RAPID_CUDA(cudaMemcpy(ids.data(), d_ids.p, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost));
    std::sort(ids.begin(), ids.end());
    *out_len = n;
    for (int32_t i = 0; i < n && i < cap; ++i) out_ids[i] = ids[(size_t)i];
    return RAPID_OK;
}

int32_t rapid_cd_aggregate(rapid_cd* cd, int64_t n_cells, const int32_t* src, const int32_t* dst, const uint8_t* ring,
                           const uint8_t* status, int64_t receiver, int32_t* out_ids, int32_t cap, int32_t* out_len) {
    (void)src;
    if (!cd || n_cells < 0 || (n_cells && (!dst || !ring || !status)) || !out_len) { set_error("bad arguments"); return RAPID_EINVAL; }
    if (!cd->raw) { set_error("rapid_cd_aggregate needs a RAPID_CD_RAW handle"); return RAPID_EINVAL; }
    if (receiver < 0 || receiver >= cd->R) { set_error("bad receiver"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    Staged st;
    RAPID_CHECK(stage_cells(cd, n_cells, dst, ring, status, nullptr, nullptr, &st));
    RAPID_CHECK(apply_common(cd, 0, n_cells, st.dst, st.ring, st.status, nullptr, DeliveryDev()));
    return take_call_marks(cd, receiver, out_ids, cap, out_len);
}

int32_t rapid_cd_invalidate(rapid_cd* cd, int64_t receiver, int32_t* out_ids, int32_t cap, int32_t* out_len) {
    if (!cd || !out_len) { set_error("bad arguments"); return RAPID_EINVAL; }
    if (!cd->raw) { set_error("rapid_cd_invalidate needs a RAPID_CD_RAW handle"); return RAPID_EINVAL; }
    if (receiver < 0 || receiver >= cd->R) { set_error("bad receiver"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    cd->last_launches = 0;
    RAPID_CHECK(ensure_id_capacity(cd));
    RAPID_CHECK(launch_sweep(cd, 0, nullptr, nullptr, DeliveryDev(), false, true));
    return take_call_marks(cd, receiver, out_ids, cap, out_len);
}

int32_t rapid_cd_get_proposal(const rapid_cd* cd, int64_t receiver, int32_t* out_ids, int32_t cap, int32_t* out_len) {
    if (!cd || !out_len || receiver < 0 || receiver >= cd->R) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    RAPID_CHECK(cd_wait(cd, false));     // clear() and asynchronous batches are still in flight on the handle's stream
    uint32_t flags = 0;
    RAPID_CUDA(cudaMemcpy(&flags, cd->rflags.p + receiver, sizeof(flags), cudaMemcpyDeviceToHost));
    *out_len = 0;
    if (!(flags & RF_ANNOUNCED) || cd->S == 0) return RAPID_OK;
    DevBuf<int32_t> d_ids, d_cnt;
    DevBuf<int64_t> d_keys;
    const int32_t S = cd->S;
    RAPID_CHECK(d_ids.reserve((size_t)S));
    RAPID_CHECK(d_keys.reserve((size_t)S));
    RAPID_CHECK(d_cnt.reserve(1));
    RAPID_CUDA(cudaMemsetAsync(d_cnt.p, 0, sizeof(int32_t), cd->stream));
    k_gather_proposal<<<(unsigned)ceil_div<int32_t>(S, 256), 256, 0, cd->stream>>>(
        rowref(cd), emit_plane(cd), S, receiver, cd->H, (1u << cd->K) - 1u, (flags & RF_RULE_GE_H) ? 1 : 0, cd->slot_subject.p, cd->view->key.p /* ring 0 row */,
        d_ids.p, d_keys.p, S, d_cnt.p);
    RAPID_KERNEL_CHECK();
    int32_t n = 0;
    RAPID_CUDA(cudaMemcpyAsync(&n, d_cnt.p, sizeof(int32_t), cudaMemcpyDeviceToHost, cd->stream));
    RAPID_CUDA(cudaStreamSynchronize(cd->stream));
    std::vector<int32_t> ids((size_t)n);
    std::vector<int64_t> keys((size_t)n);
    if (n) {
        RAPID_CUDA(cudaMemcpy(ids.data(), d_ids.p, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost));
        RAPID_CUDA(cudaMemcpy(keys.data(), d_keys.p, (size_t)n * sizeof(int64_t), cudaMemcpyDeviceToHost));
    }
    std::vector<int32_t> order((size_t)n);
    for (int32_t i = 0; i < n; ++i) order[(size_t)i] = i;
    // sorted(membershipView.getRingZeroComparator())  MembershipService.java:346-348 (signed key; id breaks exact ties)
    std::sort(order.begin(), order.end(), [&](int32_t a, int32_t b) {
        return keys[(size_t)a] != keys[(size_t)b] ? keys[(size_t)a] < keys[(size_t)b] : ids[(size_t)a] < ids[(size_t)b];
    });
    *out_len = n;
    for (int32_t i = 0; i < n && i < cap; ++i) out_ids[i] = ids[(size_t)order[(size_t)i]];
    return RAPID_OK;
}

int32_t rapid_cd_num_proposals(const rapid_cd* cd, int64_t receiver, int32_t* out) {
    if (!cd || !out || receiver < 0 || receiver >= cd->R) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    RAPID_CHECK(cd_wait(cd, false));     // clear() and asynchronous batches are still in flight on the handle's stream
    if (cd->bucketed) return replay_num_proposals(const_cast<rapid_cd*>(cd), receiver, out);
    RAPID_CUDA(cudaMemcpy(out, cd->n_prop.p + receiver, sizeof(int32_t), cudaMemcpyDeviceToHost));
    return RAPID_OK;
}

int32_t rapid_cd_debug_masks(const rapid_cd* cd, int64_t receiver, int32_t* out_subject_ids, uint16_t* out_masks, int32_t cap, int32_t* out_n) {
    if (!cd || !out_n || receiver < 0 || receiver >= cd->R) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    RAPID_CHECK(cd_wait(cd, false));     // clear() and asynchronous batches are still in flight on the handle's stream
    const int32_t S = cd->S;
    *out_n = S;
    if (S == 0) return RAPID_OK;
    DevBuf<int32_t> d_ids;
    DevBuf<uint16_t> d_m;
    RAPID_CHECK(d_ids.reserve((size_t)S));
    RAPID_CHECK(d_m.reserve((size_t)S));
    k_dump_masks<<<(unsigned)ceil_div<int32_t>(S, 256), 256, 0, cd->stream>>>(rowref(cd), S, receiver, (1u << cd->K) - 1u, cd->slot_subject.p, d_ids.p, d_m.p);
    RAPID_KERNEL_CHECK();
    const int32_t n = std::min(S, cap);
    if (out_subject_ids) RAPID_CUDA(cudaMemcpyAsync(out_subject_ids, d_ids.p, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, cd->stream));
    if (out_masks) RAPID_CUDA(cudaMemcpyAsync(out_masks, d_m.p, (size_t)n * sizeof(uint16_t), cudaMemcpyDeviceToHost, cd->stream));
    RAPID_CUDA(cudaStreamSynchronize(cd->stream));
    return RAPID_OK;
}

int32_t rapid_cd_debug_counters(const rapid_cd* cd, int64_t receiver, int32_t* updates_in_progress, int32_t* seen_link_down) {
    if (!cd || receiver < 0 || receiver >= cd->R) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    RAPID_CHECK(cd_wait(cd, false));     // clear() and asynchronous batches are still in flight on the handle's stream
    if (updates_in_progress) RAPID_CUDA(cudaMemcpy(updates_in_progress, cd->n_pre.p + receiver, sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (seen_link_down) {
        uint32_t f = 0;
        RAPID_CUDA(cudaMemcpy(&f, cd->rflags.p + receiver, sizeof(f), cudaMemcpyDeviceToHost));
        *seen_link_down = (f & RF_SEEN_DOWN) ? 1 : 0;
    }
    return RAPID_OK;
}

int32_t rapid_cd_debug_stats(const rapid_cd* cd, int32_t* n_mixed, int32_t* n_inval_pairs, int32_t* n_batch_subjects,
                             int32_t* n_valid_cells) {
    if (!cd) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    RAPID_CHECK(cd_wait(cd, false));     // clear() and asynchronous batches are still in flight on the handle's stream
    const BatchCounts& bc = cd->last;     // snapshot taken by the last kernel of the last batch
    if (n_mixed) *n_mixed = bc.n_mixed;
    if (n_batch_subjects) *n_batch_subjects = bc.n_batch_subj;
    if (n_valid_cells) *n_valid_cells = bc.n_valid;
    if (n_inval_pairs) *n_inval_pairs = cd->bucketed ? bc.n_pairs : 0;
    return RAPID_OK;
}

int32_t rapid_cd_debug_grid(const rapid_cd* cd, int32_t* apply_chunks, int32_t* prepare_blocks) {
    if (!cd) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    RAPID_CHECK(cd_wait(cd, false));
    if (apply_chunks) *apply_chunks = cd->bucketed ? cd->last_chunks : 0;
    if (prepare_blocks) *prepare_blocks = cd->last_prep_grid;
    return RAPID_OK;
}

int32_t rapid_cd_last_path(const rapid_cd* cd, int32_t* path, int32_t* n_kernel_launches) {
    if (!cd) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    RAPID_CHECK(cd_wait(cd, false));
    if (path) *path = cd->last_path;
    if (n_kernel_launches) *n_kernel_launches = cd->last_launches;
    return RAPID_OK;
}

int32_t rapid_cd_last_device_ms(const rapid_cd* cd, float* total_ms, float* main_kernel_ms) {
    if (!cd) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(cd->device);
    RAPID_CHECK(cd_wait(cd, false));
    if (total_ms) *total_ms = cd->last_ms;
    if (main_kernel_ms) *main_kernel_ms = cd->last_main_ms;
    return RAPID_OK;
}

}  // extern "C"
