// Batch preparation in ONE cooperative kernel launch, TWO grid-wide barriers (it was eight phases / seven barriers with ordered
// prefix sums; every barrier costs a grid-wide round trip plus the phase's dependent-load latency, replicated on every GPU of a sharded run):
//
//   P1  filter every alert cell (MembershipService.java:644-675); a subject without a slot is claimed by ONE of its cells
//       (compare-and-swap on slot_of) which allocates the next slot from the device counter — slot numbers are arbitrary
//       (no consumer depends on their order), so no prefix sum over "new subjects per block" is needed
//                                                                                           ── grid.sync
//   P2  cell -> slot; the cell's position among its subject's cells (atomic counter) drops its index into the subject's
//       64-entry BIN (cells beyond 64 of one subject in one call go to a shared overflow list); the first cell to touch a
//       subject in this batch gives it its index in the batch.  Also: which observers of a subject are subjects themselves
//       (refreshed when the dictionary grew) — the invalidation work list's edge table
//                                                                                           ── grid.sync
//   P3  per batch subject: its cells back into arrival order (a handful: sorted in registers), a segment of the sorted cell
//       arrays (atomic cursor), the descriptor the apply kernels consume (ring mask, first-occurrence ring sequence with
//       moments, the fresh-subject answers, fingerprint mixes)
//
// A batch has ~10 cells per subject, so bins replace the counting sort (prefix over slots + scatter) the regrouping used before.
#include <cooperative_groups.h>

#include <algorithm>
#include <climits>
#include <cstdlib>

#include "cd_internal.cuh"

namespace cg = cooperative_groups;

namespace rapid {

constexpr int PREP_THREADS = 256;

struct PrepArgs {
    int64_t A;
    const int32_t* dst;
    const uint8_t* ring;
    const uint8_t* status;
    const int64_t* cell_cfg;
    int64_t cfg;
    int raw, K, L, H;
    int64_t n_members, n_total;
    int32_t S_old, serial;   // S_old < 0: read it from bc->n_slots (bucketed handles keep it on the device)
    int32_t S_cap;           // slots the handle can hold (bucketed); a batch that needs more is rolled back (bc->overflow)
    WorkList wl;             // invalidation work list (bucketed): refreshed here whenever a subject gets a slot
    const int32_t* obs;      // view: [id][K]
    int32_t* slot_of;
    int32_t* slot_subject;
    int32_t* touch;
    int32_t* cell_slot;
    BatchCounts* bc;
    int32_t* ctr;            // [2] scratch counters: segment cursor, overflow-list length
    int regroup;
    PrepOut po;
    const int64_t* batch_off;     // sequences of batches: [n_batches + 1] cell offsets (device), else nullptr
    int32_t n_batches, seq_last;
};

// exclusive scan of one int per thread across the block; returns the thread's offset, *total = block sum
__device__ __forceinline__ int32_t block_excl_scan(int32_t v, int32_t* warp_sums, int32_t* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int32_t x = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += x;
    }
    __syncthreads();                                   // warp_sums may still be read from a previous call
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        int32_t s = lane < (PREP_THREADS >> 5) ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int32_t x = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += x;
        }
        if (lane < (PREP_THREADS >> 5)) warp_sums[lane] = s;
    }
    __syncthreads();
    *total = warp_sums[(PREP_THREADS >> 5) - 1];
    return (wid ? warp_sums[wid - 1] : 0) + inc - v;
}

__device__ __forceinline__ int32_t block_sum_before(const int32_t* arr, int upto, int32_t* warp_sums) {
    // sum of arr[0 .. upto) computed by the whole block
    int32_t s = 0;
    for (int i = threadIdx.x; i < upto; i += blockDim.x) s += arr[i];
    int32_t total;
    block_excl_scan(s, warp_sums, &total);
    return total;
}

// batch b holds the cells [batch_off[b], batch_off[b+1]): index of the batch of cell i (empty batches are skipped over)
__device__ __forceinline__ int32_t batch_of_cell(const int64_t* __restrict__ off, int32_t n_batches, int64_t i) {
    int32_t lo = 0, hi = n_batches;                 // invariant: off[lo] <= i < off[hi]
    while (hi - lo > 1) {
        const int32_t mid = (lo + hi) >> 1;
        if (off[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}

constexpr int PREP_BIN = 64;          // cells of one subject kept in its bin; the rest of a (duplicate-heavy) subject overflow
constexpr int PREP_REG = 32;          // ... of which this many are sorted in registers (~K cells per subject and batch; a few more with
                                     // re-sent duplicates or when a whole sequence of batches is prepared at once)

__global__ void __launch_bounds__(PREP_THREADS) k_prepare(PrepArgs a) {
    cg::grid_group grid = cg::this_grid();
    __shared__ int32_t warp_sums[PREP_THREADS / 32];
    __shared__ int32_t s_base;
    const int t = threadIdx.x, G = gridDim.x, bid = blockIdx.x;
    // slots in use before this batch: the host's number (sweep handles) or the device's (bucketed handles keep it on the
    // device: bc->S_before == bc->n_slots between batches — nobody writes S_before while this kernel runs)
    if (a.S_old < 0) a.S_old = a.bc->S_before;
    if (bid == 0 && t == 0) { a.ctr[0] = 0; a.ctr[1] = 0; }               // segment cursor, overflow-list length (used from P2 on)
    const int64_t gtid = (int64_t)bid * PREP_THREADS + t, gthreads = (int64_t)G * PREP_THREADS;

    // ---- P1: validity; subjects without a slot get one ---------------------------------------------------------------------
    // (counters shared by the whole grid are bumped once per block and loop iteration — thousands of same-address atomics
    // serialise in L2 — with an in-block scan handing out the individual values)
    for (int64_t i0 = (int64_t)bid * PREP_THREADS; i0 < a.A; i0 += gthreads) {
        const int64_t i = i0 + t;
        bool claimed = false;
        int32_t d = -1;
        if (i < a.A) {
            d = a.dst[i];
            int32_t v = -2;
            if (a.ring[i] >= a.K) { atomicMax(&a.bc->bad_ring, (int32_t)i); v = -1; }
            if (d < 0 || d >= a.n_total) { atomicMax(&a.bc->bad_dst, (int32_t)i); v = -1; }
            if (v == -2 && !a.raw) {
                const bool present = d < a.n_members;                         // isHostPresent
                const int st = a.status[i];
                if (a.cell_cfg && a.cell_cfg[i] != a.cfg) v = -1;              // :653
                else if (st == RAPID_EDGE_UP && present) v = -1;               // :660-665
                else if (st == RAPID_EDGE_DOWN && !present) v = -1;            // :666-671
                else if (st != RAPID_EDGE_UP && st != RAPID_EDGE_DOWN) v = -1;
            }
            a.cell_slot[i] = v;
            if (v == -2) {
                const int32_t bt = a.batch_off ? batch_of_cell(a.batch_off, a.n_batches, i) : 0;
                if (a.batch_off) a.po.cell_batch[i] = bt;             // (P3 walks a subject's cells one after the other: no searches there)
                if (a.status[i] == RAPID_EDGE_DOWN) {
                    a.bc->any_down = 1;
                    if (a.batch_off) atomicMin(&a.bc->seq_down, bt + 1);
                }
                // this cell names the subject's slot if it wins the claim
                claimed = *(volatile int32_t*)&a.slot_of[d] == -1 && atomicCAS(&a.slot_of[d], -1, -2) == -1;
            }
        }
        int32_t total;
        const int32_t off = block_excl_scan(claimed ? 1 : 0, warp_sums, &total);
        if (total) {
            if (t == 0) s_base = atomicAdd(&a.bc->n_slots, total);
            __syncthreads();
            if (claimed) {
                const int32_t slot = s_base + off;
                a.slot_subject[slot] = d;                                  // (slot < distinct ids <= capacity of the id-indexed arrays)
                a.slot_of[d] = slot;
            }
        }
    }
    grid.sync();
    const int32_t S_new = *(volatile int32_t*)&a.bc->n_slots;
    if (S_new > a.S_cap) {
        // More subjects than the handle has rows for: undo the slot assignment of this batch and apply NOTHING (the host
        // grows the handle and replays the batch; an asynchronous caller gets RAPID_ENOMEM at its next synchronisation).
        for (int64_t sl = a.S_old + gtid; sl < S_new; sl += gthreads) a.slot_of[a.slot_subject[sl]] = -1;
        grid.sync();
        if (bid == 0 && t == 0) { a.bc->overflow = 1; a.bc->need_slots = S_new; a.bc->n_slots = a.S_old; }
        return;
    }
    if (bid == 0 && t == 0) { a.bc->need_slots = S_new; a.bc->S_before = a.S_old; a.bc->seq_last = a.seq_last; }
    // ---- P2: cell -> slot, the subject's bin, distinct subjects of the batch -----------------------------------------------------
    {
        int32_t nvalid = 0;
        for (int64_t i0 = (int64_t)bid * PREP_THREADS; i0 < a.A; i0 += gthreads) {
            const int64_t i = i0 + t;
            bool first = false;
            int32_t slot = -1;
            if (i < a.A && a.cell_slot[i] == -2) {
                slot = a.slot_of[a.dst[i]];
                a.cell_slot[i] = slot;
                ++nvalid;
                first = atomicExch(&a.touch[slot], a.serial) != a.serial;   // first cell to touch the subject in this batch
                if (a.regroup) {
                    const int32_t pos = atomicAdd(&a.po.seg_cnt[slot], 1);
                    if (pos < PREP_BIN) a.po.bins[(size_t)slot * PREP_BIN + pos] = (int32_t)i;
                    else a.po.ovf[atomicAdd(&a.ctr[1], 1)] = (int32_t)i;
                }
            }
            int32_t total;
            const int32_t off = block_excl_scan(first ? 1 : 0, warp_sums, &total);
            if (total) {
                if (t == 0) s_base = atomicAdd(&a.bc->n_batch_subj, total);
                __syncthreads();
                if (first && a.regroup) { const int32_t b = s_base + off; a.po.batch_index[slot] = b; a.po.batch_slots[b] = slot; }
            }
        }
        int32_t total;
        block_excl_scan(nvalid, warp_sums, &total);
        if (t == 0 && total) atomicAdd(&a.bc->n_valid, total);
    }
    if (!a.regroup) return;
    if (a.wl.has_so && S_new > a.S_old) {
        // Some subject got a slot: refresh "which observers of this subject are subjects themselves" for every slot.  Only
        // subjects with such an observer can ever receive an implicit report (MultiNodeCutDetector.java:147-158), so only
        // they go on the invalidation work list.
        for (int64_t sl = gtid; sl < S_new; sl += gthreads) {
            const int32_t subject = a.slot_subject[sl];
            bool any = false;
            // all K observer ids, then all K slot lookups, in flight together (one loop of load -> load -> store per ring serialises
            // 2K dependent round trips: the stores may alias the tables as far as the compiler knows)
            int32_t o[RAPID_MAX_K], so[RAPID_MAX_K];
#pragma unroll
            for (int k = 0; k < RAPID_MAX_K; ++k) o[k] = k < a.K ? a.obs[(size_t)subject * a.K + k] : -1;
#pragma unroll
            for (int k = 0; k < RAPID_MAX_K; ++k) so[k] = o[k] >= 0 ? a.slot_of[o[k]] : -1;
#pragma unroll
            for (int k = 0; k < RAPID_MAX_K; ++k) {
                if (k >= a.K) break;
                a.wl.so_tab[(size_t)sl * SO_STRIDE + k] = so[k];
                if (so[k] >= 0) any = true;
            }
            const bool old = sl < a.S_old && a.wl.has_so[sl];
            a.wl.has_so[sl] = any ? 1 : 0;
            if (any && !old && sl < a.S_old) {
                // an observer of an OLDER subject joined the dictionary: the subject may sit in the unstable band of any tile
                for (int tile = 0; tile < a.wl.n_tiles; ++tile) worklist_note(a.wl, (int)tile, (int32_t)sl);
            }
        }
    }
    grid.sync();
    // ---- P3: per subject: arrival order, segment, descriptor -------------------------------------------------------------------
    const int32_t Sb = *(volatile int32_t*)&a.bc->n_batch_subj;
    const int32_t n_ovf = *(volatile int32_t*)&a.ctr[1];
    for (int64_t b0 = (int64_t)bid * PREP_THREADS; b0 < Sb; b0 += gthreads) {
        const int64_t b = b0 + t;
        const bool on = b < Sb;
        int32_t slot = -1, len = 0;
        if (on) {
            slot = a.po.batch_slots[b];
            len = a.po.seg_cnt[slot];
            a.po.seg_cnt[slot] = 0;                                        // all zero again for the next batch
        }
        int32_t total;
        const int32_t off = block_excl_scan(len, warp_sums, &total);        // the block's subjects get consecutive segments
        if (t == 0) s_base = atomicAdd(&a.ctr[0], total);
        __syncthreads();
        if (!on) continue;
        const int32_t seg_begin = s_base + off;
        int32_t* seg = a.po.sidx + seg_begin;
        SubjDesc d;
        d.slot = slot; d.bmask = 0; d.nr = 0; d.any_down = 0; d.tLf = 0; d.tHf = 0;
        d.pmask = 0; d.pdown = 0; d.pad0_ = 0; d.f_bLp = 0; d.f_bHp = 0; d.pseg_len = 0; d.pad1_ = 0;
        SubjWalk w, pw;
        int pn = 0, cf = 0;                                                // distinct rings of the prefix / of prefix + last batch
        auto take = [&](int32_t e, int32_t c, int k, uint8_t st, int32_t bt) {   // the subject's e-th cell in arrival order: ring, status, batch
            seg[e] = c;
            a.po.s_ring[seg_begin + e] = (uint8_t)k;
            a.po.s_status[seg_begin + e] = st;
            if (a.batch_off) {
                if (bt < a.seq_last) {                                     // a cell of the prefix (batches before the last one)
                    ++d.pseg_len;
                    if (st == RAPID_EDGE_DOWN) d.pdown = 1;
                    if (!((d.pmask >> k) & 1)) {
                        d.pmask |= (uint16_t)(1u << k);
                        pw.ring[pn] = (uint8_t)k;
                        pw.time[pn] = (uint32_t)bt + 1u;
                        ++pn; ++cf;
                        if (pn == a.L) d.f_bLp = (uint32_t)bt + 1u;
                        if (pn == a.H) d.f_bHp = (uint32_t)bt + 1u;
                    }
                    return;
                }
            }
            if (st == RAPID_EDGE_DOWN) d.any_down = 1;
            if (!((d.bmask >> k) & 1)) {
                d.bmask |= (uint16_t)(1u << k);
                w.ring[d.nr] = (uint8_t)k;
                w.time[d.nr] = (uint32_t)c + 1u;           // moments are 1-based cell indices (0 = "before the batch")
                ++d.nr;
                if (!((d.pmask >> k) & 1)) {               // the fresh-subject answers: its state before this batch is pmask
                    ++cf;
                    if (cf == a.L) d.tLf = (uint32_t)c + 1u;
                    if (cf == a.H) d.tHf = (uint32_t)c + 1u;
                }
            }
        };
        if (len <= PREP_REG) {
            int32_t c[PREP_REG];
#pragma unroll
            for (int q = 0; q < PREP_REG; ++q) c[q] = q < len ? a.po.bins[(size_t)slot * PREP_BIN + q] : INT_MAX;
            // insertion sort by compare-exchange on registers (fully unrolled: no local memory)
#pragma unroll
            for (int i = 1; i < PREP_REG; ++i) {
#pragma unroll
                for (int j = i; j > 0; --j) {
                    const int32_t lo = min(c[j - 1], c[j]), hi = max(c[j - 1], c[j]);
                    c[j - 1] = lo; c[j] = hi;
                }
            }
            // ring / status / batch of the cells in flight together, 16 at a time (the stores inside take() would serialise one load
            // per cell; more than 16 at once costs too many registers)
#pragma unroll
            for (int h = 0; h < PREP_REG; h += 16) {
                if (h >= len) break;
                int rk[16];
                uint8_t rs[16];
                int32_t rb[16];
#pragma unroll
                for (int q = 0; q < 16; ++q) {
                    rk[q] = h + q < len ? a.ring[c[h + q]] : 0; rs[q] = h + q < len ? a.status[c[h + q]] : 0;
                    rb[q] = (a.batch_off && h + q < len) ? a.po.cell_batch[c[h + q]] : 0;
                }
#pragma unroll
                for (int q = 0; q < 16; ++q) if (h + q < len) take(h + q, c[h + q], rk[q], rs[q], rb[q]);
            }
        } else if (len <= PREP_BIN) {
            // more cells than the register path holds (streams with re-sent duplicates; sequences of batches): sorted in the
            // thread's local memory (L1) — sorting in place in global memory cost a global-memory round trip per dependent access
            int32_t c[PREP_BIN];
            for (int q = 0; q < len; ++q) c[q] = a.po.bins[(size_t)slot * PREP_BIN + q];
            for (int i = 1; i < len; ++i) {
                const int32_t v = c[i];
                int j = i;
                for (; j > 0 && c[j - 1] > v; --j) c[j] = c[j - 1];
                c[j] = v;
            }
            uint8_t rk[PREP_BIN], rs[PREP_BIN];
            int32_t rb[PREP_BIN];
            for (int q = 0; q < len; ++q) { rk[q] = a.ring[c[q]]; rs[q] = a.status[c[q]]; rb[q] = a.batch_off ? a.po.cell_batch[c[q]] : 0; }
            for (int q = 0; q < len; ++q) take(q, c[q], rk[q], rs[q], rb[q]);
        } else {
            // a duplicate-heavy subject: the bin and the subject's cells on the shared overflow list, sorted in place (any length)
            for (int q = 0; q < PREP_BIN; ++q) seg[q] = a.po.bins[(size_t)slot * PREP_BIN + q];
            int32_t at = PREP_BIN;
            for (int32_t q = 0; q < n_ovf; ++q) {
                const int32_t ci = a.po.ovf[q];
                if (a.cell_slot[ci] == slot) seg[at++] = ci;
            }
            for (int32_t gap = len >> 1; gap > 0; gap >>= 1)
                for (int32_t i = gap; i < len; ++i) {
                    const int32_t v = seg[i];
                    int32_t j = i;
                    for (; j >= gap && seg[j - gap] > v; j -= gap) seg[j] = seg[j - gap];
                    seg[j] = v;
                }
            for (int32_t e = 0; e < len; ++e) { const int32_t ci = seg[e]; take(e, ci, a.ring[ci], a.status[ci], a.batch_off ? a.po.cell_batch[ci] : 0); }
        }
        for (int q = d.nr; q < 16; ++q) { w.ring[q] = 0; w.time[q] = 0; }
        const int32_t id = a.slot_subject[slot];
        d.mix1 = fp_mix1(id);
        d.mix2 = fp_mix2(id);
        d.seg_begin = (uint32_t)seg_begin + d.pseg_len;                    // prefix cells come first (batches are contiguous in cell order)
        d.seg_len = (uint32_t)len - d.pseg_len;
        a.po.desc[b] = d;
        a.po.walk[b] = w;
        if (a.batch_off) {
            for (int q = pn; q < 16; ++q) { pw.ring[q] = 0; pw.time[q] = 0; }
            a.po.pwalk[b] = pw;
        }
    }
}

int32_t prepare_batch(CD* cd, int64_t cfg, int64_t A, const int32_t* dst_dev, const uint8_t* ring_dev, const uint8_t* status_dev,
                      const int64_t* cfg_dev, const PrepOut* po, const int64_t* batch_off_dev, int32_t n_batches, int32_t seq_last) {
    cudaStream_t s = cd->stream;
    if (cd->prep_grid_max == 0) {
        int dev = 0, sms = TARGET_SMS, per = 4, coop = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k_prepare, PREP_THREADS, 0);
        if (!coop) { set_error("device lacks cooperative launch"); return RAPID_ECUDA; }
        cd->prep_grid_max = std::max(1, sms * std::max(per, 1));
    }
    int G = (int)std::max<int64_t>(1, std::min<int64_t>(cd->prep_grid_max, ceil_div<int64_t>(A, PREP_THREADS * 2)));
    if (const char* ov = getenv("RAPID_B200_PREP_GRID")) G = std::max(1, std::min(cd->prep_grid_max, atoi(ov)));   // test hook: forced grids
    cd->last_prep_grid = G;
    RAPID_CHECK(cd->scan_sums.reserve(8));
    PrepArgs a;
    a.A = A; a.dst = dst_dev; a.ring = ring_dev; a.status = status_dev; a.cell_cfg = cfg_dev; a.cfg = cfg;
    a.raw = cd->raw ? 1 : 0; a.K = cd->K; a.L = cd->L; a.H = cd->H;
    a.n_members = cd->view->n; a.n_total = cd->view->n + cd->view->nj;
    a.S_old = cd->bucketed ? -1 : cd->S; a.serial = ++cd->batch_serial;
    a.S_cap = cd->bucketed ? (int32_t)std::min<size_t>(cd->S_cap, 0x7fffffff) : INT_MAX;
    a.obs = cd->view->obs.p;
    memset(&a.wl, 0, sizeof(a.wl));
    if (po) a.wl = po->wl;
    a.slot_of = cd->slot_of.p; a.slot_subject = cd->slot_subject.p; a.touch = cd->touch.p;
    a.cell_slot = cd->cell_slot.p; a.bc = cd->counts.p;
    a.ctr = cd->scan_sums.p;
    a.regroup = po ? 1 : 0;
    a.batch_off = (po && cd->bucketed) ? batch_off_dev : nullptr; a.n_batches = n_batches; a.seq_last = a.batch_off ? seq_last : 0;
    if (po) a.po = *po; else memset(&a.po, 0, sizeof(a.po));
    void* args[] = {(void*)&a};
    RAPID_CUDA(cudaLaunchCooperativeKernel((void*)k_prepare, dim3((unsigned)G), dim3(PREP_THREADS), args, 0, s));
    cd->last_launches += 1;
    return RAPID_OK;
}

}  // namespace rapid
