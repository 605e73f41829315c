// Alert generation on the device (SURVEY.md §8 f4): the K ping-pong edge failure detectors of every virtual node
// (PingPongFailureDetector.java:38-121, one per entry of getSubjectsOf(myAddr), MembershipService.java:697-707) and the
// AlertMessages their notifiers raise (edgeFailureNotification, MembershipService.java:472-495), as cells ready for
// rapid_cd_apply_batch_dev.  One 32-bit word per detector; one tick = one failure-detector interval of the whole cluster:
// a single elementwise pass (HBM-bound: 4-8 B of state + 4 B of subject table per detector); the few detectors that notify are
// appended to a list, sorted back into detector order, and expanded into alerts and cells.
#include <limits.h>


#include <vector>

#include "common.cuh"
#include "radix.cuh"
#include "scan.cuh"
#include "wire_internal.cuh"

namespace rapid {

// detector word: bits 0..22 failureCount, bit 23 notified, bits 24..31 bootstrapResponseCount (saturating; only "> 30" is read)
#define FD_CNT_MASK 0x7fffffu
#define FD_NOTIFIED (1u << 23)

struct FdScal {
    int32_t n_fired;                    // detectors whose notifier fired in this interval
    int32_t n_cells;                    // ring numbers of their AlertMessages
};

// One interval: run() of every detector (:75-85).  A detector that notifies appends its index to `fired` (rare: the list
// is sorted afterwards, so the atomics' order does not matter); a quiet interval touches nothing but the state words.
__global__ void k_fd_tick(uint32_t D, uint32_t K, const int32_t* __restrict__ subj, const uint8_t* __restrict__ flags,
                          const uint8_t* __restrict__ edge_fail, int32_t thr, int32_t boot_thr, uint32_t* __restrict__ st,
                          uint32_t* __restrict__ fired, FdScal* __restrict__ sc) {
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= D) return;
    const uint32_t o = idx / K;                                                  // 32-bit: D < 2^31 is checked at create
    const uint8_t fo = flags[o];
    if (fo & RAPID_FD_CRASHED) return;                                           // a crashed process runs nothing
    uint32_t w = st[idx];
    if ((int32_t)(w & FD_CNT_MASK) >= thr && !(w & FD_NOTIFIED)) {               // hasFailed() && !notified (:76-79)
        st[idx] = w | FD_NOTIFIED;
        fired[atomicAdd(&sc->n_fired, 1)] = idx;
        return;
    }
    const uint32_t w0 = w;                                                       // probe (:80-84) and its callback
    const uint8_t fs = flags[subj[idx]];
    const bool fail = (edge_fail && edge_fail[idx]) || (fo & RAPID_FD_EGRESS_BLOCKED) || (fs & (RAPID_FD_CRASHED | RAPID_FD_INGRESS_BLOCKED));
    bool count = fail;
    if (!fail && (fs & RAPID_FD_BOOTSTRAPPING)) {                                // :97-104
        uint32_t b = w >> 24;
        if (b < 255) ++b;
        w = (w & 0x00ffffffu) | (b << 24);
        count = (int32_t)b > boot_thr;
    }
    if (count && (w & FD_CNT_MASK) < FD_CNT_MASK) w = (w & ~FD_CNT_MASK) | ((w & FD_CNT_MASK) + 1);   // :120-123
    if (w != w0) st[idx] = w;                                                    // healthy edges write nothing
}

// number of ring numbers of each fired detector's AlertMessage: getRingNumbers(myAddr, subject) (MembershipView.java:397-418)
__global__ void k_fd_count(int32_t nf, uint32_t K, const uint32_t* __restrict__ fired_sorted, const int32_t* __restrict__ subj,
                           int32_t* __restrict__ cnt) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nf) return;
    const uint32_t idx = fired_sorted[i], o = idx / K;
    const int32_t s = subj[idx];
    int c = 0;
    for (uint32_t r = 0; r < K; ++r) c += subj[o * K + r] == s ? 1 : 0;
    cnt[i] = c;
}

// alerts and cells of the detectors that fired, in detector order (node, then ring of the detector), rings ascending
__global__ void k_fd_emit(int32_t nf, uint32_t K, const uint32_t* __restrict__ fired_sorted, const int32_t* __restrict__ subj,
                          const int32_t* __restrict__ cnt, const int32_t* __restrict__ pos, int64_t cfg, int32_t* __restrict__ a_obs,
                          int32_t* __restrict__ a_subj, uint16_t* __restrict__ a_mask, int32_t* __restrict__ c_src,
                          int32_t* __restrict__ c_dst, uint8_t* __restrict__ c_ring, uint8_t* __restrict__ c_status,
                          int64_t* __restrict__ c_cfg, FdScal* __restrict__ sc) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nf) return;
    if (i == nf - 1) sc->n_cells = pos[i] + cnt[i];
    const uint32_t idx = fired_sorted[i], o = idx / K;
    const int32_t s = subj[idx];
    int32_t c = pos[i];
    uint32_t mask = 0;
    for (uint32_t r = 0; r < K; ++r) {
        if (subj[o * K + r] != s) continue;
        mask |= 1u << r;
        c_src[c] = (int32_t)o; c_dst[c] = s; c_ring[c] = (uint8_t)r; c_status[c] = RAPID_EDGE_DOWN; c_cfg[c] = cfg;
        ++c;
    }
    a_obs[i] = (int32_t)o; a_subj[i] = s; a_mask[i] = (uint16_t)mask;
}
__global__ void k_fd_begin(FdScal* sc) { sc->n_fired = 0; sc->n_cells = 0; }

// ---- join and leave alerts merged into the interval (rapid_fdet_merge_alerts) ----------------------------------------------------
// ids[0 .. nj) are the listed joiners, ids[nj .. nj + nl) the listed leavers; the rows of both are obs[id][K] (a joiner's expected
// observers, a member's getObserversOf).  Candidate m < nf is the tick's alert m; candidate nf + i * K + k is observer k of ids[i],
// so the candidates are laid out [tick | joins * K | leaves * K].  A joiner raises one alert per distinct live observer (its first
// ring); a leaver one per live observer and ring, repeats kept (MembershipService.leave sends one LeaveMessage per entry of
// getObserversOf).  Sort key = (sender << mb) | candidate, candidate < 2^mb: per sender, the tick's alerts first in their order,
// then the join alerts, then the leave alerts, each in list order.  A dropped candidate gets all ones, above every kept key.
__global__ void k_fd_merge_keys(int64_t M, int32_t nf, uint32_t K, int64_t nj, int mb, const int32_t* __restrict__ a_obs,
                                const int32_t* __restrict__ ids, const int32_t* __restrict__ obs_tab, const uint8_t* __restrict__ flags,
                                uint64_t* __restrict__ key, FdScal* __restrict__ sc) {
    const int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    int32_t o;
    bool keep = true;
    if (m < nf) {
        o = a_obs[m];
    } else {
        const int64_t s = m - nf, i = s / K;
        const uint32_t k = (uint32_t)(s - i * K);
        const int32_t* row = obs_tab + (int64_t)ids[i] * K;
        o = row[k];
        if (i < nj)                                                              // a joiner's observer sends once, on its first ring
            for (uint32_t q = 0; q < k; ++q) keep &= row[q] != o;
        keep &= !(flags[o] & RAPID_FD_CRASHED);                                  // a crashed observer sends nothing
    }
    key[m] = keep ? (((uint64_t)(uint32_t)o << mb) | (uint64_t)m) : ~0ull;
    if (keep) atomicAdd(&sc->n_fired, 1);
}
// ring numbers of every kept alert, in merged order: {r : obs[id][r] == sender} for a join or leave alert
__global__ void k_fd_merge_count(int32_t nv, int32_t nf, uint32_t K, int mb, const uint64_t* __restrict__ skey, const uint16_t* __restrict__ a_mask,
                                 const int32_t* __restrict__ ids, const int32_t* __restrict__ obs_tab, uint16_t* __restrict__ mask,
                                 int32_t* __restrict__ cnt) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nv) return;
    const int64_t m = (int64_t)(skey[i] & ((1ull << mb) - 1));
    uint32_t mk;
    if (m < nf) {
        mk = a_mask[m];
    } else {
        const int64_t s = m - nf, j = s / K;
        const int32_t* row = obs_tab + (int64_t)ids[j] * K;
        const int32_t o = (int32_t)(skey[i] >> mb);
        mk = 0;
        for (uint32_t r = 0; r < K; ++r) mk |= (row[r] == o ? 1u : 0u) << r;
    }
    mask[i] = (uint16_t)mk;
    cnt[i] = __popc(mk);
}
__global__ void k_fd_merge_emit(int32_t nv, int32_t nf, uint32_t K, int64_t nj, int mb, const uint64_t* __restrict__ skey,
                                const int32_t* __restrict__ a_subj, const int32_t* __restrict__ ids, const uint16_t* __restrict__ mask,
                                const int32_t* __restrict__ cnt, const int32_t* __restrict__ pos, int64_t tick_cfg, int64_t merge_cfg,
                                int32_t* __restrict__ o_obs, int32_t* __restrict__ o_subj, int32_t* __restrict__ c_src,
                                int32_t* __restrict__ c_dst, uint8_t* __restrict__ c_ring, uint8_t* __restrict__ c_status,
                                int64_t* __restrict__ c_cfg, FdScal* __restrict__ sc) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nv) return;
    if (i == nv - 1) sc->n_cells = pos[i] + cnt[i];
    const int64_t m = (int64_t)(skey[i] & ((1ull << mb) - 1));
    const int32_t o = (int32_t)(skey[i] >> mb);
    const bool tick = m < nf;
    const int64_t j = tick ? 0 : (m - nf) / K;
    const int32_t s = tick ? a_subj[m] : ids[j];
    const uint8_t st = (!tick && j < nj) ? RAPID_EDGE_UP : RAPID_EDGE_DOWN;
    const int64_t cc = tick ? tick_cfg : merge_cfg;
    const uint32_t mk = mask[i];
    int32_t c = pos[i];
    for (uint32_t r = 0; r < K; ++r) {
        if (!((mk >> r) & 1u)) continue;
        c_src[c] = o; c_dst[c] = s; c_ring[c] = (uint8_t)r; c_status[c] = st; c_cfg[c] = cc;
        ++c;
    }
    o_obs[i] = o; o_subj[i] = s;
}

struct FD {
    const View* view = nullptr;
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    float last_ms = 0.f;
    int64_t n = 0;
    int K = 0;
    int32_t thr = 10, boot_thr = 30;
    uint64_t view_epoch = 0;
    DevBuf<uint32_t> st, fired, fired_sorted;
    DevBuf<int32_t> cnt, pos;
    DevBuf<uint8_t> flags, edge;
    DevBuf<int32_t> scan_sums;
    RadixScratch rs;
    DevBuf<FdScal> sc;
    PinnedBuf<FdScal> h_sc;
    int64_t n_alerts = 0, n_cells = 0;
    DevBuf<int32_t> a_obs, a_subj, c_src, c_dst;
    DevBuf<uint16_t> a_mask;
    DevBuf<uint8_t> c_ring, c_status;
    DevBuf<int64_t> c_cfg;
    // the last tick's node flags / configuration (merged alerts skip crashed observers of that interval), and the merge's buffers
    const uint8_t* tick_flags = nullptr;
    int64_t tick_cfg = 0;
    bool merged = false;                   // join / leave alerts were merged into this interval already
    DevBuf<int32_t> j_ids, m_obs, m_subj, m_src, m_dst;
    DevBuf<uint64_t> j_key, j_skey;
    DevBuf<uint16_t> m_mask;
    DevBuf<uint8_t> m_ring, m_status;
    DevBuf<int64_t> m_cfg;
};

template <typename T>
static void swap_buf(DevBuf<T>& a, DevBuf<T>& b) { std::swap(a.p, b.p); std::swap(a.cap, b.cap); }

static const int TB = 256;
static inline unsigned grid_for(int64_t n) { return (unsigned)ceil_div<int64_t>(n > 0 ? n : 1, TB); }

static int32_t fd_alloc(FD* fd) {
    const View* v = fd->view;
    fd->n = v->n; fd->K = v->K; fd->view_epoch = v->member_epoch;
    const size_t D = (size_t)std::max<int64_t>(fd->n * fd->K, 1);
    if (fd->n * fd->K > 0x7ffffff0LL) { set_error("more than 2^31 detectors"); return RAPID_EINVAL; }
    RAPID_CHECK(fd->st.reserve(D)); RAPID_CHECK(fd->fired.reserve(D));      // at most every detector fires in one interval
    RAPID_CHECK(fd->flags.reserve((size_t)std::max<int64_t>(fd->n, 1))); RAPID_CHECK(fd->edge.reserve(D));
    RAPID_CUDA(cudaMemsetAsync(fd->st.p, 0, D * sizeof(uint32_t), fd->stream));
    fd->n_alerts = fd->n_cells = 0;
    fd->tick_flags = nullptr;
    return RAPID_OK;
}

static int32_t fd_read_scal(FD* fd) {
    RAPID_CUDA(cudaMemcpyAsync(fd->h_sc.p, fd->sc.p, sizeof(FdScal), cudaMemcpyDeviceToHost, fd->stream));
    RAPID_CUDA(cudaStreamSynchronize(fd->stream));
    return RAPID_OK;
}

static int32_t fd_tick_device(FD* fd, const uint8_t* d_flags, const uint8_t* d_edge, int64_t cfg, int64_t* n_alerts, int64_t* n_cells) {
    cudaStream_t s = fd->stream;
    const int64_t D = fd->n * fd->K;
    fd->n_alerts = fd->n_cells = 0;
    fd->tick_flags = d_flags; fd->tick_cfg = cfg; fd->merged = false;
    if (fd->n >= 2 && D > 0) {                               // getSubjectsOf is empty in a one-node view (MembershipView.java:270-272)
        k_fd_begin<<<1, 1, 0, s>>>(fd->sc.p);
        k_fd_tick<<<grid_for(D), TB, 0, s>>>((uint32_t)D, (uint32_t)fd->K, fd->view->subj.p, d_flags, d_edge, fd->thr, fd->boot_thr, fd->st.p,
                                             fd->fired.p, fd->sc.p);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(fd_read_scal(fd));                       // a quiet interval ends here: one kernel, one 8-byte readback
        const int32_t nf = fd->h_sc.p->n_fired;
        if (nf > 0) {
            const size_t F = (size_t)nf, C = F * (size_t)fd->K;      // a fired detector yields at most K cells
            RAPID_CHECK(fd->fired_sorted.reserve(F)); RAPID_CHECK(fd->cnt.reserve(F)); RAPID_CHECK(fd->pos.reserve(F));
            RAPID_CHECK(fd->a_obs.reserve(F)); RAPID_CHECK(fd->a_subj.reserve(F)); RAPID_CHECK(fd->a_mask.reserve(F));
            RAPID_CHECK(fd->c_src.reserve(C)); RAPID_CHECK(fd->c_dst.reserve(C)); RAPID_CHECK(fd->c_ring.reserve(C));
            RAPID_CHECK(fd->c_status.reserve(C)); RAPID_CHECK(fd->c_cfg.reserve(C));
            // the notifying detectors back into (node, detector) order: hand-written radix sort (radix.cuh), keys only
            RAPID_CHECK(radix_sort_pairs<uint32_t>(fd->rs, fd->fired.p, nullptr, fd->fired_sorted.p, nullptr, nf, 0, 32, s, false));
            k_fd_count<<<grid_for(nf), TB, 0, s>>>(nf, (uint32_t)fd->K, fd->fired_sorted.p, fd->view->subj.p, fd->cnt.p);
            RAPID_KERNEL_CHECK();
            RAPID_CHECK(exclusive_scan_i32_to(fd->cnt.p, fd->pos.p, nf, fd->scan_sums, s));
            k_fd_emit<<<grid_for(nf), TB, 0, s>>>(nf, (uint32_t)fd->K, fd->fired_sorted.p, fd->view->subj.p, fd->cnt.p, fd->pos.p, cfg, fd->a_obs.p,
                                                 fd->a_subj.p, fd->a_mask.p, fd->c_src.p, fd->c_dst.p, fd->c_ring.p, fd->c_status.p, fd->c_cfg.p, fd->sc.p);
            RAPID_KERNEL_CHECK();
            RAPID_CHECK(fd_read_scal(fd));
            fd->n_alerts = nf; fd->n_cells = fd->h_sc.p->n_cells;
        }
    }
    if (n_alerts) *n_alerts = fd->n_alerts;
    if (n_cells) *n_cells = fd->n_cells;
    return RAPID_OK;
}

}  // namespace rapid

using namespace rapid;

struct rapid_fdet : rapid::FD {};

void rapid::fdet_interval_dev(const rapid_fdet* fd, FdetInterval* out) {
    out->view = fd->view; out->device = fd->device;
    out->have = fd->tick_flags != nullptr && fd->view_epoch == fd->view->member_epoch && fd->n == fd->view->n;
    out->n_alerts = fd->n_alerts;
    out->obs = fd->a_obs.p; out->subj = fd->a_subj.p; out->mask = fd->a_mask.p;
    out->cell_status = fd->c_status.p; out->cell_cfg = fd->c_cfg.p;
}

extern "C" {

int32_t rapid_fdet_create(rapid_fdet** out, const rapid_view* v, int32_t failure_threshold, int32_t bootstrap_threshold) {
    if (!out || !v || failure_threshold < 1 || failure_threshold > 1000000 || bootstrap_threshold < 0 || bootstrap_threshold > 254) { set_error("bad arguments"); return RAPID_EINVAL; }
    *out = nullptr;
    DeviceGuard g(v->device);
    rapid_fdet* fd = new rapid_fdet();
    fd->view = v; fd->device = v->device; fd->thr = failure_threshold; fd->boot_thr = bootstrap_threshold;
    int32_t rc = RAPID_OK;
    do {
        if (cudaStreamCreateWithFlags(&fd->stream, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreate(&fd->ev0) != cudaSuccess ||
            cudaEventCreate(&fd->ev1) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "stream", __FILE__, __LINE__); break; }
        if ((rc = fd->sc.reserve(1)) || (rc = fd->h_sc.reserve(1))) break;
        if ((rc = fd_alloc(fd))) break;
        if (cudaStreamSynchronize(fd->stream) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "init", __FILE__, __LINE__); break; }
    } while (0);
    if (rc) { rapid_fdet_destroy(fd); return rc; }
    *out = fd;
    return RAPID_OK;
}

int32_t rapid_fdet_destroy(rapid_fdet* h) {
    rapid_fdet* fd = h;
    if (!fd) return RAPID_OK;
    DeviceGuard g(fd->device);
    if (fd->stream) { cudaStreamSynchronize(fd->stream); cudaStreamDestroy(fd->stream); }
    if (fd->ev0) cudaEventDestroy(fd->ev0);
    if (fd->ev1) cudaEventDestroy(fd->ev1);
    delete fd;
    return RAPID_OK;
}

int32_t rapid_fdet_reset(rapid_fdet* h) {
    rapid_fdet* fd = h;
    if (!fd) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(fd->device);
    return fd_alloc(fd);
}

int32_t rapid_fdet_tick(rapid_fdet* h, const uint8_t* node_flags, const uint8_t* edge_fail, int64_t cfg_id, int64_t* n_alerts, int64_t* n_cells) {
    rapid_fdet* fd = h;
    if (!fd || (fd->n && !node_flags)) { set_error("bad arguments"); return RAPID_EINVAL; }
    if (fd->view_epoch != fd->view->member_epoch || fd->n != fd->view->n) { set_error("the view changed: call rapid_fdet_reset (detectors are re-created per configuration)"); return RAPID_EINVAL; }
    DeviceGuard g(fd->device);
    cudaStream_t s = fd->stream;
    RAPID_CUDA(cudaEventRecord(fd->ev0, s));
    if (fd->n) RAPID_CUDA(cudaMemcpyAsync(fd->flags.p, node_flags, (size_t)fd->n, cudaMemcpyHostToDevice, s));
    if (edge_fail && fd->n) RAPID_CUDA(cudaMemcpyAsync(fd->edge.p, edge_fail, (size_t)(fd->n * fd->K), cudaMemcpyHostToDevice, s));
    const int32_t rc = fd_tick_device(fd, fd->flags.p, edge_fail ? fd->edge.p : nullptr, cfg_id, n_alerts, n_cells);
    if (rc == RAPID_OK) { cudaEventRecord(fd->ev1, s); cudaEventSynchronize(fd->ev1); cudaEventElapsedTime(&fd->last_ms, fd->ev0, fd->ev1); }
    return rc;
}

int32_t rapid_fdet_tick_dev(rapid_fdet* h, const uint8_t* node_flags_dev, const uint8_t* edge_fail_dev, int64_t cfg_id, int64_t* n_alerts,
                            int64_t* n_cells) {
    rapid_fdet* fd = h;
    if (!fd || (fd->n && !node_flags_dev)) { set_error("bad arguments"); return RAPID_EINVAL; }
    if (fd->view_epoch != fd->view->member_epoch || fd->n != fd->view->n) { set_error("the view changed: call rapid_fdet_reset"); return RAPID_EINVAL; }
    DeviceGuard g(fd->device);
    cudaStream_t s = fd->stream;
    RAPID_CUDA(cudaEventRecord(fd->ev0, s));
    const int32_t rc = fd_tick_device(fd, node_flags_dev, edge_fail_dev, cfg_id, n_alerts, n_cells);
    if (rc == RAPID_OK) { cudaEventRecord(fd->ev1, s); cudaEventSynchronize(fd->ev1); cudaEventElapsedTime(&fd->last_ms, fd->ev0, fd->ev1); }
    return rc;
}

int32_t rapid_fdet_cells_dev(const rapid_fdet* h, const int32_t** src, const int32_t** dst, const uint8_t** ring, const uint8_t** status,
                             const int64_t** cfg) {
    const rapid_fdet* fd = h;
    if (!fd) { set_error("NULL handle"); return RAPID_EINVAL; }
    if (src) *src = fd->c_src.p;
    if (dst) *dst = fd->c_dst.p;
    if (ring) *ring = fd->c_ring.p;
    if (status) *status = fd->c_status.p;
    if (cfg) *cfg = fd->c_cfg.p;
    return RAPID_OK;
}

// The interval's cells grouped the way the reference ships them: AlertBatcher (MembershipService.java:613-637) sends ONE
// BatchedAlertMessage per sender and window, so batch b = the cells raised by one observer (cells are ordered by node already).
// batch_off[0 .. *n_batches] for rapid_cd_apply_batches[_dev]; RAPID_ENOMEM if cap (entries) is too small (*n_batches is set).
int32_t rapid_fdet_sender_batches(const rapid_fdet* h, int64_t* batch_off, int64_t cap, int64_t* n_batches) {
    const rapid_fdet* fd = h;
    if (!fd || !n_batches || (cap > 0 && !batch_off)) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(fd->device);
    const size_t n = (size_t)fd->n_cells;
    std::vector<int32_t> src(n);
    if (n) {
        RAPID_CUDA(cudaMemcpyAsync(src.data(), fd->c_src.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, fd->stream));
        RAPID_CUDA(cudaStreamSynchronize(fd->stream));
    }
    int64_t nb = 0;
    for (size_t i = 0; i < n; ++i) {
        if (i == 0 || src[i] != src[i - 1]) { if (nb < cap) batch_off[nb] = (int64_t)i; ++nb; }
    }
    *n_batches = nb;
    if (nb + 1 > cap) { set_error("batch_off holds %lld entries, %lld needed", (long long)cap, (long long)nb + 1); return RAPID_ENOMEM; }
    batch_off[nb] = (int64_t)n;
    return RAPID_OK;
}

int32_t rapid_fdet_merge_alerts(rapid_fdet* h, const int32_t* joiner_ids, int64_t n_joiners, const int32_t* leaver_ids, int64_t n_leavers,
                                int64_t cfg_id, int64_t* n_alerts, int64_t* n_cells) {
    rapid_fdet* fd = h;
    if (!fd || n_joiners < 0 || (n_joiners && !joiner_ids) || n_leavers < 0 || (n_leavers && !leaver_ids)) { set_error("bad arguments"); return RAPID_EINVAL; }
    if (fd->view_epoch != fd->view->member_epoch || fd->n != fd->view->n) { set_error("the view changed: call rapid_fdet_reset"); return RAPID_EINVAL; }
    if (!fd->tick_flags) { set_error("no interval to add join alerts to (call rapid_fdet_tick first)"); return RAPID_EINVAL; }
    // the merged list no longer tells the tick's alerts from merged ones: a second merge would turn earlier UP alerts into DOWN ones
    if (fd->merged) { set_error("join alerts were already added to this interval (one call per tick)"); return RAPID_EINVAL; }
    const View* v = fd->view;
    for (int64_t i = 0; i < n_joiners; ++i)
        if (joiner_ids[i] < v->n || joiner_ids[i] >= v->n + v->nj) { set_error("id %d is not a registered joiner", joiner_ids[i]); return RAPID_EINVAL; }
    for (int64_t i = 0; i < n_leavers; ++i)
        if (leaver_ids[i] < 0 || leaver_ids[i] >= v->n) { set_error("id %d is not a member", leaver_ids[i]); return RAPID_EINVAL; }
    const int64_t nl = fd->n >= 2 ? n_leavers : 0;          // getObserversOf is empty in a one-node view (MembershipView.java:240-242)
    const int64_t nf = fd->n_alerts, lim = 1LL << 30;
    if (n_joiners >= lim || nl >= lim || nf + (n_joiners + nl) * fd->K >= lim) {
        set_error("too many %s alerts in one interval", n_leavers ? "join and leave" : "join"); return RAPID_EINVAL;
    }
    const int64_t nj = n_joiners, ni = nj + nl, M = nf + ni * fd->K;
    DeviceGuard g(fd->device);
    cudaStream_t s = fd->stream;
    const uint32_t K = (uint32_t)fd->K;
    fd->last_ms = 0.f;
    if (ni > 0) {
        RAPID_CUDA(cudaEventRecord(fd->ev0, s));
        RAPID_CHECK(fd->j_ids.reserve((size_t)ni)); RAPID_CHECK(fd->j_key.reserve((size_t)M)); RAPID_CHECK(fd->j_skey.reserve((size_t)M));
        if (nj) RAPID_CUDA(cudaMemcpyAsync(fd->j_ids.p, joiner_ids, (size_t)nj * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        if (nl) RAPID_CUDA(cudaMemcpyAsync(fd->j_ids.p + nj, leaver_ids, (size_t)nl * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        k_fd_begin<<<1, 1, 0, s>>>(fd->sc.p);
        int mb = 1;                                                              // candidates are < 2^mb
        while ((1LL << mb) < M) ++mb;
        k_fd_merge_keys<<<grid_for(M), TB, 0, s>>>(M, (int32_t)nf, K, nj, mb, fd->a_obs.p, fd->j_ids.p, v->obs.p, fd->tick_flags, fd->j_key.p, fd->sc.p);
        RAPID_KERNEL_CHECK();
        int ob = 1;                                                              // senders are member ids < 2^ob
        while ((1LL << ob) <= fd->n) ++ob;
        RAPID_CHECK(radix_sort_pairs<uint64_t>(fd->rs, fd->j_key.p, nullptr, fd->j_skey.p, nullptr, M, 0, mb + ob, s, true));
        RAPID_CHECK(fd_read_scal(fd));
        const int32_t nv = fd->h_sc.p->n_fired;                                 // kept: the tick's alerts + the merged ones
        if (nv > nf) {
            const size_t F = (size_t)nv, C = F * K;
            RAPID_CHECK(fd->cnt.reserve(F)); RAPID_CHECK(fd->pos.reserve(F)); RAPID_CHECK(fd->m_mask.reserve(F));
            RAPID_CHECK(fd->m_obs.reserve(F)); RAPID_CHECK(fd->m_subj.reserve(F));
            RAPID_CHECK(fd->m_src.reserve(C)); RAPID_CHECK(fd->m_dst.reserve(C)); RAPID_CHECK(fd->m_ring.reserve(C));
            RAPID_CHECK(fd->m_status.reserve(C)); RAPID_CHECK(fd->m_cfg.reserve(C));
            k_fd_merge_count<<<grid_for(nv), TB, 0, s>>>(nv, (int32_t)nf, K, mb, fd->j_skey.p, fd->a_mask.p, fd->j_ids.p, v->obs.p, fd->m_mask.p, fd->cnt.p);
            RAPID_KERNEL_CHECK();
            RAPID_CHECK(exclusive_scan_i32_to(fd->cnt.p, fd->pos.p, nv, fd->scan_sums, s));
            // the merged interval is written beside the tick's (it reads them), then takes their place
            k_fd_merge_emit<<<grid_for(nv), TB, 0, s>>>(nv, (int32_t)nf, K, nj, mb, fd->j_skey.p, fd->a_subj.p, fd->j_ids.p, fd->m_mask.p, fd->cnt.p,
                                                       fd->pos.p, fd->tick_cfg, cfg_id, fd->m_obs.p, fd->m_subj.p, fd->m_src.p, fd->m_dst.p,
                                                       fd->m_ring.p, fd->m_status.p, fd->m_cfg.p, fd->sc.p);
            RAPID_KERNEL_CHECK();
            RAPID_CHECK(fd_read_scal(fd));
            swap_buf(fd->a_obs, fd->m_obs); swap_buf(fd->a_subj, fd->m_subj); swap_buf(fd->a_mask, fd->m_mask);
            swap_buf(fd->c_src, fd->m_src); swap_buf(fd->c_dst, fd->m_dst); swap_buf(fd->c_ring, fd->m_ring);
            swap_buf(fd->c_status, fd->m_status); swap_buf(fd->c_cfg, fd->m_cfg);
            fd->n_alerts = nv; fd->n_cells = fd->h_sc.p->n_cells;
        }
        RAPID_CUDA(cudaEventRecord(fd->ev1, s));
        RAPID_CUDA(cudaEventSynchronize(fd->ev1));
        RAPID_CUDA(cudaEventElapsedTime(&fd->last_ms, fd->ev0, fd->ev1));
    }
    fd->merged = true;
    if (n_alerts) *n_alerts = fd->n_alerts;
    if (n_cells) *n_cells = fd->n_cells;
    return RAPID_OK;
}

int32_t rapid_fdet_join_alerts(rapid_fdet* h, const int32_t* joiner_ids, int64_t n, int64_t cfg_id, int64_t* n_alerts, int64_t* n_cells) {
    return rapid_fdet_merge_alerts(h, joiner_ids, n, nullptr, 0, cfg_id, n_alerts, n_cells);
}

int32_t rapid_fdet_read_cells(const rapid_fdet* h, int32_t* src, int32_t* dst, uint8_t* ring, uint8_t* status, int64_t* cfg) {
    const rapid_fdet* fd = h;
    if (!fd) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(fd->device);
    const size_t n = (size_t)fd->n_cells;
    if (n == 0) return RAPID_OK;
    cudaStream_t s = fd->stream;
    if (src) RAPID_CUDA(cudaMemcpyAsync(src, fd->c_src.p, n * 4, cudaMemcpyDeviceToHost, s));
    if (dst) RAPID_CUDA(cudaMemcpyAsync(dst, fd->c_dst.p, n * 4, cudaMemcpyDeviceToHost, s));
    if (ring) RAPID_CUDA(cudaMemcpyAsync(ring, fd->c_ring.p, n, cudaMemcpyDeviceToHost, s));
    if (status) RAPID_CUDA(cudaMemcpyAsync(status, fd->c_status.p, n, cudaMemcpyDeviceToHost, s));
    if (cfg) RAPID_CUDA(cudaMemcpyAsync(cfg, fd->c_cfg.p, n * 8, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

int32_t rapid_fdet_read_alerts(const rapid_fdet* h, int32_t* observer, int32_t* subject, uint16_t* ring_mask) {
    const rapid_fdet* fd = h;
    if (!fd) { set_error("NULL handle"); return RAPID_EINVAL; }
    DeviceGuard g(fd->device);
    const size_t n = (size_t)fd->n_alerts;
    if (n == 0) return RAPID_OK;
    cudaStream_t s = fd->stream;
    if (observer) RAPID_CUDA(cudaMemcpyAsync(observer, fd->a_obs.p, n * 4, cudaMemcpyDeviceToHost, s));
    if (subject) RAPID_CUDA(cudaMemcpyAsync(subject, fd->a_subj.p, n * 4, cudaMemcpyDeviceToHost, s));
    if (ring_mask) RAPID_CUDA(cudaMemcpyAsync(ring_mask, fd->a_mask.p, n * 2, cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

int32_t rapid_fdet_state(const rapid_fdet* h, int64_t node, int32_t k, int32_t* failure_count, int32_t* notified) {
    const rapid_fdet* fd = h;
    if (!fd || node < 0 || node >= fd->n || k < 0 || k >= fd->K) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(fd->device);
    uint32_t w = 0;
    RAPID_CUDA(cudaStreamSynchronize(fd->stream));
    RAPID_CUDA(cudaMemcpy(&w, fd->st.p + node * fd->K + k, sizeof(uint32_t), cudaMemcpyDeviceToHost));
    if (failure_count) *failure_count = (int32_t)(w & FD_CNT_MASK);
    if (notified) *notified = (w & FD_NOTIFIED) ? 1 : 0;
    return RAPID_OK;
}

int32_t rapid_fdet_last_device_ms(const rapid_fdet* h, float* total_ms) {
    const rapid_fdet* fd = h;
    if (!fd || !total_ms) return RAPID_EINVAL;
    *total_ms = fd->last_ms;
    return RAPID_OK;
}

}  // extern "C"
