// MembershipView on the device: K rings as structure-of-arrays in HBM.
//
// Follows rapid/src/main/java/com/vrg/rapid/MembershipView.java:
//   ring k  = members sorted by signed key  xx_k(hostname)*31 + xx_k.hashInt(port)        (:562-587)
//   observers = ring successors (:234-257), subjects / expected observers = predecessors (:308-322)
//   configuration id = 37-ary polynomial hash over identifiersSeen then ring-0 order       (:544-556)
// Not a port: the Java keeps K red-black trees of Endpoint objects with a memoised comparator; here every
// (ring, node) key is hashed in one kernel, each ring is one radix sort (radix.cuh), and the observer/subject relations
// become two dense int32 tables that the cut-detection kernels index directly.
#include <algorithm>
#include <string>
#include <vector>

#include "common.cuh"
#include "radix.cuh"
#include "scan.cuh"

namespace rapid {

// ------------------------------------------------------------------ kernels
__global__ void k_ring_keys(const uint8_t* __restrict__ hb, const int32_t* __restrict__ off,
                            const int32_t* __restrict__ port, int64_t first, int64_t count, int K,
                            int64_t* __restrict__ key, size_t stride) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count * K) return;
    const int k = (int)(t / count);
    const int64_t i = first + t % count;
    const int32_t o = off[i];
    key[(size_t)k * stride + i] = ring_key(hb + o, off[i + 1] - o, port[i], k);
}

// sortable unsigned image of a signed key
__global__ void k_flip_keys(const int64_t* __restrict__ key, size_t stride, int k, int64_t n,
                            uint64_t* __restrict__ ukey, int32_t* __restrict__ ids) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ukey[i] = (uint64_t)key[(size_t)k * stride + i] ^ 0x8000000000000000ULL;
    ids[i] = (int32_t)i;
}

__global__ void k_unflip_and_check(const uint64_t* __restrict__ ukey_sorted, int64_t n, int64_t* __restrict__ sorted_key,
                                   int32_t* __restrict__ collision /* [2]: position, ring */, int k) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    sorted_key[i] = (int64_t)(ukey_sorted[i] ^ 0x8000000000000000ULL);
    if (i + 1 < n && ukey_sorted[i] == ukey_sorted[i + 1]) {
        if (atomicCAS(&collision[0], -1, (int32_t)i) == -1) collision[1] = k;
    }
}

__global__ void k_tables(const int32_t* __restrict__ ring, int64_t n, int K, int32_t* __restrict__ obs,
                         int32_t* __restrict__ subj, int32_t* __restrict__ pos0) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * K) return;
    const int k = (int)(t / n);
    const int64_t p = t % n;
    const int32_t* r = ring + (size_t)k * n;
    const int32_t node = r[p];
    if (n <= 1) {
        obs[(size_t)node * K + k] = -1;
        subj[(size_t)node * K + k] = -1;
    } else {
        obs[(size_t)node * K + k] = r[p + 1 == n ? 0 : p + 1];        // TreeSet.higher, wrap to first()
        subj[(size_t)node * K + k] = r[p == 0 ? n - 1 : p - 1];       // TreeSet.lower, wrap to last()
    }
    if (k == 0) pos0[node] = (int32_t)p;
}

// Joiners: expected observers = predecessor of the joiner's key on every ring (getExpectedObserversOf :292-303).
// flag[j] = 1 if the identical endpoint is already a member.
__global__ void k_joiner_rows(const uint8_t* __restrict__ hb, const int32_t* __restrict__ off,
                              const int32_t* __restrict__ port, const int64_t* __restrict__ key, size_t stride,
                              const int64_t* __restrict__ sorted_key, const int32_t* __restrict__ ring, int64_t n,
                              int K, int64_t first, int64_t count, int32_t* __restrict__ obs, int32_t* __restrict__ flag) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count * K) return;
    const int k = (int)(t / count);
    const int64_t id = first + t % count;
    const int64_t kj = key[(size_t)k * stride + id];
    const int64_t* sk = sorted_key + (size_t)k * n;
    // lower_bound: first position with sk[pos] >= kj
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (sk[mid] < kj) lo = mid + 1; else hi = mid;
    }
    int32_t pred = -1;
    if (n > 0) pred = ring[(size_t)k * n + (lo == 0 ? n - 1 : lo - 1)];
    obs[(size_t)id * K + k] = pred;
    if (k == 0 && lo < n && sk[lo] == kj) {
        const int32_t m = ring[lo];
        const int32_t oa = off[id], ob = off[m];
        const int32_t la = off[id + 1] - oa, lb = off[m + 1] - ob;
        bool same = (la == lb) && (port[id] == port[m]);
        for (int32_t c = 0; same && c < la; ++c) same = hb[oa + c] == hb[ob + c];
        if (same) flag[t % count] = 1;
    }
}

// Configuration id: hash = 1; for x in X: hash = hash*37 + x  (wrapping).  X = hashLong(high),hashLong(low) of the
// sorted identifiers, then xx0(hostname), xx0.hashInt(port) in ring-0 order.
__device__ __forceinline__ uint64_t pow37(uint64_t e) {
    uint64_t r = 1, b = 37;
    while (e) { if (e & 1) r *= b; b *= b; e >>= 1; }
    return r;
}

__global__ void k_config_id(const int64_t* __restrict__ id_high, const int64_t* __restrict__ id_low,
                            const int32_t* __restrict__ id_order, int64_t n_ids, const uint8_t* __restrict__ hb,
                            const int32_t* __restrict__ off, const int32_t* __restrict__ port,
                            const int32_t* __restrict__ ring0, int64_t n, unsigned long long* __restrict__ out) {
    const int64_t M = 2 * n_ids + 2 * n;
    const int SEG = 32;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t s = t * SEG;
    uint64_t h = 0;
    if (s < M) {
        const int64_t e = (s + SEG < M) ? s + SEG : M;
        for (int64_t i = s; i < e; ++i) {
            uint64_t x;
            if (i < 2 * n_ids) {
                const int32_t j = id_order ? id_order[i >> 1] : (int32_t)(i >> 1);
                x = xxh64_long((i & 1) ? id_low[j] : id_high[j], 0);
            } else {
                const int64_t q = i - 2 * n_ids;
                const int32_t node = ring0[q >> 1];
                if (q & 1) x = xxh64_int(port[node], 0);
                else { const int32_t o = off[node]; x = xxh64_bytes(hb + o, off[node + 1] - o, 0); }
            }
            h = h * 37 + x;
        }
        h *= pow37((uint64_t)(M - e));
        if (t == 0) h += pow37((uint64_t)M);     // the leading "hash = 1"
    } else if (t == 0) {
        h = 1;                                    // M == 0
    }
    // block reduce (wrapping add)
    __shared__ unsigned long long sm[32];
    unsigned long long v = h;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
        v = threadIdx.x < (blockDim.x + 31) / 32 ? sm[threadIdx.x] : 0ULL;
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (threadIdx.x == 0 && v) atomicAdd(out, v);
    }
}

__global__ void k_id_sort_keys(const int64_t* __restrict__ v, int64_t n, uint64_t* __restrict__ out, int32_t* idx,
                               const int32_t* __restrict__ order_in) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t j = order_in ? order_in[i] : (int32_t)i;
    out[i] = (uint64_t)v[j] ^ 0x8000000000000000ULL;
    idx[i] = j;
}

// ------------------------------------------------------------------ host helpers
struct CutScratch {                                      // rapid_view_apply_cut: everything it builds beside the live arrays
    DevBuf<int32_t> d_cut, incut, newid, kept, len, err, map, flag, pos, jv, jv2, collision, off2, port2, ring2;
    DevBuf<uint64_t> jk, jk2;
    DevBuf<uint8_t> hb2;
    DevBuf<int64_t> key2, sk2, nhi2, nlo2;
};
struct IdScratch {                                       // NodeId sorting / merging
    DevBuf<uint64_t> k_in, k_out;
    DevBuf<int32_t> i_in, i_mid, order, dup;
    DevBuf<int64_t> bh, bl, oh, ol;
};
struct ViewScratch {
    RadixScratch rs;
    DevBuf<int32_t> scan_sums;
    CutScratch cut;
    IdScratch ids;
};
static ViewScratch* scratch(View* v) {
    if (!v->scratch) v->scratch = new ViewScratch();
    return static_cast<ViewScratch*>(v->scratch);
}

// (keys_in, vals_in) are scratch for the caller: the sort may use them as its ping-pong buffers
static int32_t sort_pairs(View* v, uint64_t* kin, uint64_t* kout, int32_t* vin, int32_t* vout, int64_t n, cudaStream_t s) {
    return radix_sort_pairs<uint64_t>(scratch(v)->rs, kin, vin, kout, vout, n, 0, 64, s);
}

static int32_t ensure_total_capacity(View* v, int64_t ntot) {
    if ((size_t)ntot <= v->key_stride) return RAPID_OK;
    size_t ns = v->key_stride ? v->key_stride : 1;
    while (ns < (size_t)ntot) ns *= 2;
    DevBuf<int64_t> nk;
    RAPID_CHECK(nk.reserve(ns * (size_t)v->K));
    if (v->key.p && v->key_stride) {
        RAPID_CUDA(cudaMemcpy2DAsync(nk.p, ns * sizeof(int64_t), v->key.p, v->key_stride * sizeof(int64_t),
                                     (size_t)(v->n + v->nj) * sizeof(int64_t), (size_t)v->K, cudaMemcpyDeviceToDevice,
                                     v->stream));
        RAPID_CUDA(cudaStreamSynchronize(v->stream));
    }
    std::swap(v->key.p, nk.p);
    std::swap(v->key.cap, nk.cap);
    v->key_stride = ns;
    RAPID_CHECK(v->obs.reserve(ns * (size_t)v->K, true, v->stream));
    return RAPID_OK;
}

// Append `count` endpoints after the ones the view holds (members then joiners).  The endpoint table lives on the device only:
// hostname bytes, offsets and ports are appended in place (no host mirror).  *added_bytes lets a failed caller undo it.
static int32_t upload_endpoints(View* v, int64_t count, const uint8_t* hb, const int32_t* off, const int32_t* port, size_t* added_bytes = nullptr) {
    const int64_t base = v->n + v->nj;      // v->n must already be set for members (0 during create)
    const size_t old_bytes = v->host_bytes_len;
    const size_t add_bytes = count ? (size_t)(off[count] - off[0]) : 0;
    std::vector<int32_t> rebased((size_t)count + 1);
    rebased[0] = (int32_t)old_bytes;
    for (int64_t i = 0; i < count; ++i) {
        const int32_t len = off[i + 1] - off[i];
        if (len < 0) { set_error("host_off must be non-decreasing"); return RAPID_EINVAL; }
        rebased[(size_t)i + 1] = rebased[(size_t)i] + len;
    }
    if (old_bytes + add_bytes > 0x7fffffffULL) { set_error("hostname bytes exceed 2 GiB"); return RAPID_EINVAL; }
    RAPID_CHECK(v->host_bytes.reserve(std::max<size_t>(1, old_bytes + add_bytes), true, v->stream));
    RAPID_CHECK(v->host_off.reserve((size_t)(base + count + 1), true, v->stream));
    RAPID_CHECK(v->port.reserve(std::max<size_t>(1, (size_t)(base + count)), true, v->stream));
    if (add_bytes)
        RAPID_CUDA(cudaMemcpyAsync(v->host_bytes.p + old_bytes, hb + off[0], add_bytes, cudaMemcpyHostToDevice, v->stream));
    RAPID_CUDA(cudaMemcpyAsync(v->host_off.p + base, rebased.data(), (size_t)(count + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, v->stream));
    if (count)
        RAPID_CUDA(cudaMemcpyAsync(v->port.p + base, port, (size_t)count * sizeof(int32_t), cudaMemcpyHostToDevice, v->stream));
    RAPID_CUDA(cudaStreamSynchronize(v->stream));
    v->host_bytes_len = old_bytes + add_bytes;
    if (added_bytes) *added_bytes = add_bytes;
    return RAPID_OK;
}

// error reporting only: are the endpoints with ids a and b of a device endpoint table the same (hostname, port)?
static bool same_endpoint(const uint8_t* hb, const int32_t* off, const int32_t* port, int64_t a, int64_t b) {
    int32_t oa[2], ob[2], pa = 0, pb = 0;
    if (cudaMemcpy(oa, off + a, sizeof(oa), cudaMemcpyDeviceToHost) != cudaSuccess) return false;
    if (cudaMemcpy(ob, off + b, sizeof(ob), cudaMemcpyDeviceToHost) != cudaSuccess) return false;
    cudaMemcpy(&pa, port + a, sizeof(pa), cudaMemcpyDeviceToHost);
    cudaMemcpy(&pb, port + b, sizeof(pb), cudaMemcpyDeviceToHost);
    const int32_t la = oa[1] - oa[0], lb = ob[1] - ob[0];
    if (la != lb || pa != pb) return false;
    std::vector<uint8_t> ba((size_t)std::max(la, 1)), bb((size_t)std::max(lb, 1));
    if (la) { cudaMemcpy(ba.data(), hb + oa[0], (size_t)la, cudaMemcpyDeviceToHost); cudaMemcpy(bb.data(), hb + ob[0], (size_t)lb, cudaMemcpyDeviceToHost); }
    return memcmp(ba.data(), bb.data(), (size_t)la) == 0;
}
static bool same_endpoint(const View* v, int64_t a, int64_t b) {
    return same_endpoint(v->host_bytes.p, v->host_off.p, v->port.p, a, b);
}

static int32_t build_rings(View* v) {
    const int64_t n = v->n;
    const int K = v->K;
    cudaStream_t s = v->stream;
    RAPID_CHECK(ensure_total_capacity(v, std::max<int64_t>(n, 1)));
    RAPID_CHECK(v->sorted_key.reserve(std::max<size_t>(1, (size_t)n * K)));
    RAPID_CHECK(v->ring.reserve(std::max<size_t>(1, (size_t)n * K)));
    RAPID_CHECK(v->pos0.reserve(std::max<size_t>(1, (size_t)n)));
    RAPID_CHECK(v->subj.reserve(std::max<size_t>(1, (size_t)n * K)));
    if (n == 0) return RAPID_OK;
    const int TB = 256;
    k_ring_keys<<<(unsigned)ceil_div<int64_t>(n * K, TB), TB, 0, s>>>(v->host_bytes.p, v->host_off.p, v->port.p, 0, n, K,
                                                                      v->key.p, v->key_stride);
    RAPID_KERNEL_CHECK();
    DevBuf<uint64_t> uk_in, uk_out;
    DevBuf<int32_t> id_in, collision;
    RAPID_CHECK(uk_in.reserve((size_t)n));
    RAPID_CHECK(uk_out.reserve((size_t)n));
    RAPID_CHECK(id_in.reserve((size_t)n));
    RAPID_CHECK(collision.reserve(2));
    RAPID_CUDA(cudaMemsetAsync(collision.p, 0xff, 2 * sizeof(int32_t), s));
    for (int k = 0; k < K; ++k) {
        k_flip_keys<<<(unsigned)ceil_div<int64_t>(n, TB), TB, 0, s>>>(v->key.p, v->key_stride, k, n, uk_in.p, id_in.p);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(sort_pairs(v, uk_in.p, uk_out.p, id_in.p, v->ring.p + (size_t)k * n, n, s));
        k_unflip_and_check<<<(unsigned)ceil_div<int64_t>(n, TB), TB, 0, s>>>(uk_out.p, n, v->sorted_key.p + (size_t)k * n,
                                                                             collision.p, k);
        RAPID_KERNEL_CHECK();
    }
    int32_t coll[2];
    RAPID_CUDA(cudaMemcpyAsync(coll, collision.p, sizeof(coll), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    if (coll[0] >= 0) {
        int32_t ids[2];
        RAPID_CUDA(cudaMemcpy(ids, v->ring.p + (size_t)coll[1] * n + coll[0], sizeof(ids), cudaMemcpyDeviceToHost));
        if (same_endpoint(v, ids[0], ids[1])) {
            set_error("endpoint given twice (node ids %d and %d): NodeAlreadyInRingException", ids[0], ids[1]);
            return RAPID_EALREADY_IN_RING;
        }
        set_error("ring-%d key collision between node ids %d and %d (TreeSet would silently drop one)", coll[1], ids[0], ids[1]);
        return RAPID_EHASH_COLLISION;
    }
    k_tables<<<(unsigned)ceil_div<int64_t>(n * K, TB), TB, 0, s>>>(v->ring.p, n, K, v->obs.p, v->subj.p, v->pos0.p);
    RAPID_KERNEL_CHECK();
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

}  // namespace rapid

using namespace rapid;

extern "C" {

int32_t rapid_view_create(rapid_view** out, int32_t K, int64_t n, const uint8_t* host_bytes, const int32_t* host_off,
                          const int32_t* port, int32_t device) {
    if (!out) { set_error("out is NULL"); return RAPID_EINVAL; }
    *out = nullptr;
    if (K < 1 || K > RAPID_MAX_K) { set_error("K must be in [1, %d], got %d", RAPID_MAX_K, K); return RAPID_EINVAL; }
    if (n < 0 || n > 0x7ffffff0LL) { set_error("bad n"); return RAPID_EINVAL; }
    if (n > 0 && (!host_bytes || !host_off || !port)) { set_error("NULL endpoint arrays"); return RAPID_EINVAL; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        set_error("no CUDA device: librapid_b200 has no CPU fallback");
        return RAPID_ECUDA;
    }
    if (device < 0 || device >= ndev) { set_error("device %d out of range (%d devices)", device, ndev); return RAPID_EINVAL; }
    DeviceGuard g(device);
    rapid_view* v = new rapid_view();
    v->device = device;
    v->K = K;
    int32_t rc = RAPID_OK;
    do {
        if (cudaStreamCreateWithFlags(&v->stream, cudaStreamNonBlocking) != cudaSuccess) { rc = cuda_fail(cudaGetLastError(), "stream", __FILE__, __LINE__); break; }
        static const int32_t zero_off[1] = {0};
        rc = upload_endpoints(v, n, host_bytes, n ? host_off : zero_off, port);
        if (rc) break;
        v->n = n;
        rc = build_rings(v);
    } while (0);
    if (rc) { rapid_view_destroy(v); return rc; }
    *out = v;
    return RAPID_OK;
}

int32_t rapid_view_destroy(rapid_view* v) {
    if (!v) return RAPID_OK;
    DeviceGuard g(v->device);
    if (v->stream) cudaStreamDestroy(v->stream);
    if (v->scratch) { delete static_cast<ViewScratch*>(v->scratch); v->scratch = nullptr; }
    delete v;
    return RAPID_OK;
}

int32_t rapid_view_size(const rapid_view* v, int64_t* out_n) {
    if (!v || !out_n) { set_error("NULL argument"); return RAPID_EINVAL; }
    *out_n = v->n;
    return RAPID_OK;
}

int32_t rapid_view_num_joiners(const rapid_view* v, int64_t* out) {
    if (!v || !out) { set_error("NULL argument"); return RAPID_EINVAL; }
    *out = v->nj;
    return RAPID_OK;
}

int32_t rapid_view_ring(const rapid_view* v, int32_t k, int32_t* out_ids) {
    if (!v || k < 0 || k >= v->K || (!out_ids && v->n)) { set_error("bad ring index %d", k); return RAPID_EINVAL; }
    DeviceGuard g(v->device);
    if (v->n) RAPID_CUDA(cudaMemcpy(out_ids, v->ring.p + (size_t)k * v->n, (size_t)v->n * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return RAPID_OK;
}

int32_t rapid_view_keys(const rapid_view* v, int32_t k, int64_t* out_keys) {
    if (!v || k < 0 || k >= v->K) { set_error("bad ring index %d", k); return RAPID_EINVAL; }
    DeviceGuard g(v->device);
    const int64_t tot = v->n + v->nj;
    if (tot) RAPID_CUDA(cudaMemcpy(out_keys, v->key.p + (size_t)k * v->key_stride, (size_t)tot * sizeof(int64_t), cudaMemcpyDeviceToHost));
    return RAPID_OK;
}

static int32_t member_row(const rapid_view* v, const int32_t* table, int32_t node, int32_t* out, int32_t* out_count) {
    if (!v || !out || !out_count) { set_error("NULL argument"); return RAPID_EINVAL; }
    if (node < 0 || node >= v->n) { set_error("node %d is not in the ring", node); return RAPID_ENOT_IN_RING; }
    if (v->n <= 1) { *out_count = 0; return RAPID_OK; }
    DeviceGuard g(v->device);
    RAPID_CUDA(cudaMemcpy(out, table + (size_t)node * v->K, (size_t)v->K * sizeof(int32_t), cudaMemcpyDeviceToHost));
    *out_count = v->K;
    return RAPID_OK;
}

int32_t rapid_view_observers(const rapid_view* v, int32_t node, int32_t* out, int32_t* out_count) {
    return member_row(v, v ? v->obs.p : nullptr, node, out, out_count);
}

int32_t rapid_view_subjects(const rapid_view* v, int32_t node, int32_t* out, int32_t* out_count) {
    return member_row(v, v ? v->subj.p : nullptr, node, out, out_count);
}

int32_t rapid_view_tables(const rapid_view* v, int32_t* out_obs, int32_t* out_subj) {
    if (!v) { set_error("NULL view"); return RAPID_EINVAL; }
    DeviceGuard g(v->device);
    const size_t bytes = (size_t)v->n * v->K * sizeof(int32_t);
    if (bytes && out_obs) RAPID_CUDA(cudaMemcpy(out_obs, v->obs.p, bytes, cudaMemcpyDeviceToHost));
    if (bytes && out_subj) RAPID_CUDA(cudaMemcpy(out_subj, v->subj.p, bytes, cudaMemcpyDeviceToHost));
    return RAPID_OK;
}

int32_t rapid_view_joiner_tables(const rapid_view* v, int32_t* out) {
    if (!v || (!out && v->nj)) { set_error("NULL argument"); return RAPID_EINVAL; }
    DeviceGuard g(v->device);
    if (v->nj) RAPID_CUDA(cudaMemcpy(out, v->obs.p + (size_t)v->n * v->K, (size_t)v->nj * v->K * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return RAPID_OK;
}

int32_t rapid_view_ring_numbers(const rapid_view* v, int32_t observer, int32_t subject, uint16_t* out_mask) {
    if (!v || !out_mask) { set_error("NULL argument"); return RAPID_EINVAL; }
    int32_t row[RAPID_MAX_K], cnt = 0;
    RAPID_CHECK(rapid_view_subjects(v, observer, row, &cnt));
    uint16_t m = 0;
    for (int k = 0; k < cnt; ++k) if (row[k] == subject) m |= (uint16_t)(1u << k);
    *out_mask = m;
    return RAPID_OK;
}

// Computes joiner rows for endpoints [first, first+count) already uploaded; flags identical members.
static int32_t joiner_rows(rapid_view* v, int64_t first, int64_t count, std::vector<int32_t>& flags) {
    cudaStream_t s = v->stream;
    const int TB = 256;
    k_ring_keys<<<(unsigned)ceil_div<int64_t>(count * v->K, TB), TB, 0, s>>>(v->host_bytes.p, v->host_off.p, v->port.p, first,
                                                                             count, v->K, v->key.p, v->key_stride);
    RAPID_KERNEL_CHECK();
    DevBuf<int32_t> flag;
    RAPID_CHECK(flag.reserve((size_t)count));
    RAPID_CUDA(cudaMemsetAsync(flag.p, 0, (size_t)count * sizeof(int32_t), s));
    k_joiner_rows<<<(unsigned)ceil_div<int64_t>(count * v->K, TB), TB, 0, s>>>(
        v->host_bytes.p, v->host_off.p, v->port.p, v->key.p, v->key_stride, v->sorted_key.p, v->ring.p, v->n, v->K, first,
        count, v->obs.p, flag.p);
    RAPID_KERNEL_CHECK();
    flags.resize((size_t)count);
    RAPID_CUDA(cudaMemcpyAsync(flags.data(), flag.p, (size_t)count * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

static void pop_endpoints(rapid_view* v, size_t bytes) { v->host_bytes_len -= bytes; }     // the entries past n + nj are simply forgotten

int32_t rapid_view_register_joiners(rapid_view* v, int64_t n_add, const uint8_t* host_bytes, const int32_t* host_off,
                                    const int32_t* port, int32_t* out_first_id) {
    if (!v || n_add < 0 || (n_add && (!host_bytes || !host_off || !port))) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(v->device);
    const int64_t first = v->n + v->nj;
    if (out_first_id) *out_first_id = (int32_t)first;
    if (n_add == 0) return RAPID_OK;
    if (first + n_add > 0x7ffffff0LL) { set_error("too many endpoints"); return RAPID_EINVAL; }
    RAPID_CHECK(ensure_total_capacity(v, first + n_add));
    size_t added = 0;
    RAPID_CHECK(upload_endpoints(v, n_add, host_bytes, host_off, port, &added));
    std::vector<int32_t> flags;
    int32_t rc = joiner_rows(v, first, n_add, flags);
    if (rc == RAPID_OK) {
        for (int64_t j = 0; j < n_add; ++j)
            if (flags[(size_t)j]) { set_error("joiner %lld is already a member", (long long)j); rc = RAPID_EALREADY_IN_RING; break; }
    }
    if (rc != RAPID_OK) { pop_endpoints(v, added); return rc; }
    if (v->has_node_ids) {                                   // NodeIds of the new joiners are unknown until rapid_view_set_joiner_ids
        RAPID_CHECK(v->node_hi.reserve((size_t)(first + n_add), true, v->stream));
        RAPID_CHECK(v->node_lo.reserve((size_t)(first + n_add), true, v->stream));
        RAPID_CUDA(cudaMemsetAsync(v->node_hi.p + first, 0, (size_t)n_add * sizeof(int64_t), v->stream));
        RAPID_CUDA(cudaMemsetAsync(v->node_lo.p + first, 0, (size_t)n_add * sizeof(int64_t), v->stream));
    }
    v->nj += n_add;
    ++v->epoch;
    return RAPID_OK;
}

}  // extern "C"

namespace rapid {

// ==================================================================================================================
// decideViewChange on the device (MembershipService.java:385-444): ringDelete (:167-201) of the members in the cut,
// ringAdd (:123-160) of the joiners in it, on all K rings — as one order-preserving compaction of every ring plus one
// sorted merge of the (few) joiners into it; the endpoint table, the per-id keys and the NodeIds are compacted alongside.
// Nothing visits the host except the cut's ids (in) and two status words (out).
// ==================================================================================================================
__global__ void k_cut_mark(const int32_t* __restrict__ cut, int64_t n_cut, int64_t n, int64_t tot, int32_t* __restrict__ incut,
                           int32_t* __restrict__ err /* [0] = code (1 range, 2 twice), [1] = id */) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cut) return;
    const int32_t id = cut[i];
    if (id < 0 || id >= tot) { if (atomicCAS(&err[0], 0, 1) == 0) err[1] = id; return; }
    if (atomicExch(&incut[id], 1) != 0) { if (atomicCAS(&err[0], 0, 2) == 0) err[1] = id; }
    (void)n;
}
// members stay unless they are in the cut, joiners come in only if they are
__global__ void k_cut_keep(int64_t n, int64_t tot, const int32_t* __restrict__ incut, const int32_t* __restrict__ off,
                           int32_t* __restrict__ keep, int32_t* __restrict__ len) {
    const int64_t id = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= tot) return;
    const int k = id < n ? (incut[id] ? 0 : 1) : (incut[id] ? 1 : 0);
    keep[id] = k;
    len[id] = k ? off[id + 1] - off[id] : 0;
}
__global__ void k_cut_endpoints(int64_t tot, const int32_t* __restrict__ keep, const int32_t* __restrict__ newid,
                                const int32_t* __restrict__ newoff, const int32_t* __restrict__ off, const uint8_t* __restrict__ hb,
                                const int32_t* __restrict__ port, uint8_t* __restrict__ hb2, int32_t* __restrict__ off2,
                                int32_t* __restrict__ port2, const int64_t* __restrict__ nhi, const int64_t* __restrict__ nlo,
                                int64_t* __restrict__ nhi2, int64_t* __restrict__ nlo2, int32_t* __restrict__ map, int32_t total_bytes, int32_t n2) {
    const int64_t id = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (id == 0) off2[n2] = total_bytes;
    if (id >= tot) return;
    if (!keep[id]) { map[id] = -1; return; }
    const int32_t q = newid[id], o = off[id], o2 = newoff[id], l = off[id + 1] - o;
    map[id] = q;
    off2[q] = o2;
    port2[q] = port[id];
    for (int32_t c = 0; c < l; ++c) hb2[o2 + c] = hb[o + c];
    if (nhi) { nhi2[q] = nhi[id]; nlo2[q] = nlo[id]; }
}
__global__ void k_cut_keys(int K, int64_t tot, size_t stride, size_t stride2, const int32_t* __restrict__ keep,
                           const int32_t* __restrict__ newid, const int64_t* __restrict__ key, int64_t* __restrict__ key2) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)K * tot) return;
    const int k = (int)(t / tot);
    const int64_t id = t % tot;
    if (keep[id]) key2[(size_t)k * stride2 + newid[id]] = key[(size_t)k * stride + id];
}
__global__ void k_cut_ring_flags(int K, int64_t n, const int32_t* __restrict__ ring, const int32_t* __restrict__ keep, int32_t* __restrict__ flag) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < (int64_t)K * n) flag[t] = keep[ring[t]];
}
// the admitted joiners of every ring as (sortable key, new id) pairs: jk[k][j], jv[k][j]
__global__ void k_cut_joiner_keys(int K, int64_t n, int64_t tot, size_t stride, const int32_t* __restrict__ keep, const int32_t* __restrict__ newid,
                                  int32_t n_surv, int32_t m, const int64_t* __restrict__ key, uint64_t* __restrict__ jk, int32_t* __restrict__ jv) {
    const int64_t id = n + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int k = blockIdx.y;
    if (k >= K || id >= tot || !keep[id]) return;
    const int32_t j = newid[id] - n_surv;
    jk[(size_t)k * m + j] = (uint64_t)key[(size_t)k * stride + id] ^ 0x8000000000000000ULL;
    jv[(size_t)k * m + j] = newid[id];
}
// collision[0] = ring of the first equal-key pair found (-1: none), collision[1..2] = the pair's new ids
__device__ __forceinline__ void cut_collision(int32_t* collision, int k, int32_t a, int32_t b) {
    if (atomicCAS(&collision[0], -1, k) == -1) { collision[1] = a; collision[2] = b; }
}
// the (few) joiners of every ring sorted by key: rank = number of joiners with a smaller key, all pairs through shared memory;
// two joiners with the same key on a ring -> collision (TreeSet.add would silently drop one)
__global__ void __launch_bounds__(256) k_cut_joiner_rank(int32_t m, const uint64_t* __restrict__ jk, const int32_t* __restrict__ jv,
                                                         uint64_t* __restrict__ jk2, int32_t* __restrict__ jv2, int32_t* __restrict__ collision) {
    __shared__ uint64_t s_k[256];
    const int k = blockIdx.y;
    const uint64_t* mk = jk + (size_t)k * m;
    const int32_t* mv = jv + (size_t)k * m;
    const int32_t i = blockIdx.x * 256 + threadIdx.x;
    const uint64_t key = i < m ? mk[i] : 0ull;
    int32_t rank = 0;
    for (int32_t b = 0; b < m; b += 256) {
        __syncthreads();
        s_k[threadIdx.x] = b + (int32_t)threadIdx.x < m ? mk[b + threadIdx.x] : ~0ull;
        __syncthreads();
        const int32_t lim = min(256, m - b);
        for (int32_t j = 0; j < lim; ++j) {
            const uint64_t o = s_k[j];
            rank += o < key ? 1 : 0;
            if (o == key && b + j != i && i < m) cut_collision(collision, k, mv[i], mv[b + j]);
        }
    }
    if (i < m) { jk2[(size_t)k * m + rank] = key; jv2[(size_t)k * m + rank] = mv[i]; }
}
// after the per-ring radix sorts of the joiners: equal keys are adjacent (as k_unflip_and_check finds them for build_rings)
__global__ void k_cut_joiner_adjacent(int K, int32_t m, const uint64_t* __restrict__ jk2, const int32_t* __restrict__ jv2,
                                      int32_t* __restrict__ collision) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (int64_t)K * m) return;
    const int32_t j = (int32_t)(t % m);
    if (j + 1 < m && jk2[t] == jk2[t + 1]) cut_collision(collision, (int)(t / m), jv2[t], jv2[t + 1]);
}
// merge of every ring (blockIdx.y): survivors keep their order, every joiner slots in by its key (TreeSet order of the new membership)
__global__ void k_cut_merge(int64_t n, int32_t n_surv, int32_t m, const int32_t* __restrict__ ring, const int64_t* __restrict__ sorted_key,
                            const int32_t* __restrict__ flag, const int32_t* __restrict__ pos /* exclusive scan of flag over [K][n] */,
                            const int32_t* __restrict__ newid, const uint64_t* __restrict__ jk_all, const int32_t* __restrict__ jv_all,
                            int32_t* __restrict__ ring2, int64_t* __restrict__ sorted_key2, int32_t* __restrict__ collision) {
    const int k = blockIdx.y;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int32_t* fl = flag + (size_t)k * n;
    const int32_t* ps = pos + (size_t)k * n;
    const int64_t* sk = sorted_key + (size_t)k * n;
    const uint64_t* jk = jk_all + (size_t)k * m;
    const int32_t* jv = jv_all + (size_t)k * m;
    const int32_t base = n ? ps[0] : 0;
    const int32_t n2 = n_surv + m;
    if (t < n) {
        if (!fl[t]) return;
        const uint64_t u = (uint64_t)sk[t] ^ 0x8000000000000000ULL;
        int32_t lo = 0, hi = m;                               // joiners with a smaller key
        while (lo < hi) { const int32_t mid = (lo + hi) >> 1; if (jk[mid] < u) lo = mid + 1; else hi = mid; }
        const int32_t me = newid[ring[(size_t)k * n + t]];
        if (lo < m && jk[lo] == u) cut_collision(collision, k, me, jv[lo]);
        const int32_t out = (ps[t] - base) + lo;
        ring2[(size_t)k * n2 + out] = me;
        sorted_key2[(size_t)k * n2 + out] = sk[t];
    } else if (t < n + m) {
        const int32_t i = (int32_t)(t - n);
        const int64_t key = (int64_t)(jk[i] ^ 0x8000000000000000ULL);
        int64_t lo = 0, hi = n;                               // first old position whose key is >= the joiner's
        while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (sk[mid] < key) lo = mid + 1; else hi = mid; }
        const int32_t before = n == 0 ? 0 : (lo < n ? ps[lo] - base : ps[n - 1] + fl[n - 1] - base);
        if (lo < n && sk[lo] == key && fl[lo]) cut_collision(collision, k, jv[i], newid[ring[(size_t)k * n + lo]]);
        const int32_t out = before + i;
        ring2[(size_t)k * n2 + out] = jv[i];
        sorted_key2[(size_t)k * n2 + out] = key;
    }
}

// ---- identifiersSeen (MembershipView.java:58-60, :126-128, :474-500) ---------------------------------------------------------
__global__ void k_u64_flip(const int64_t* __restrict__ v, const int32_t* __restrict__ order, int64_t n, uint64_t* __restrict__ out, int32_t* __restrict__ idx) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t j = order ? order[i] : (int32_t)i;
    out[i] = (uint64_t)v[j] ^ 0x8000000000000000ULL;
    idx[i] = j;
}
__global__ void k_gather_ids(const int64_t* __restrict__ hi, const int64_t* __restrict__ lo, const int32_t* __restrict__ order, int64_t n,
                             int64_t* __restrict__ hi2, int64_t* __restrict__ lo2) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { hi2[i] = hi[order[i]]; lo2[i] = lo[order[i]]; }
}
// sorts n (hi, lo) pairs by signed (hi, lo) into (hi2, lo2): LSD — stable sort by low, then by high
static int32_t sort_node_ids(View* v, const int64_t* hi, const int64_t* lo, int64_t n, int64_t* hi2, int64_t* lo2) {
    if (n <= 0) return RAPID_OK;
    cudaStream_t s = v->stream;
    const int TB = 256;
    const unsigned gb = (unsigned)ceil_div<int64_t>(n, TB);
    IdScratch& c = scratch(v)->ids;
    DevBuf<uint64_t>& k_in = c.k_in; DevBuf<uint64_t>& k_out = c.k_out;
    DevBuf<int32_t>& i_in = c.i_in; DevBuf<int32_t>& i_mid = c.i_mid; DevBuf<int32_t>& order = c.order;
    RAPID_CHECK(k_in.reserve((size_t)n)); RAPID_CHECK(k_out.reserve((size_t)n));
    RAPID_CHECK(i_in.reserve((size_t)n)); RAPID_CHECK(i_mid.reserve((size_t)n)); RAPID_CHECK(order.reserve((size_t)n));
    k_u64_flip<<<gb, TB, 0, s>>>(lo, nullptr, n, k_in.p, i_in.p);
    RAPID_KERNEL_CHECK();
    RAPID_CHECK(sort_pairs(v, k_in.p, k_out.p, i_in.p, i_mid.p, n, s));
    k_u64_flip<<<gb, TB, 0, s>>>(hi, i_mid.p, n, k_in.p, i_in.p);
    RAPID_KERNEL_CHECK();
    RAPID_CHECK(sort_pairs(v, k_in.p, k_out.p, i_in.p, order.p, n, s));
    k_gather_ids<<<gb, TB, 0, s>>>(hi, lo, order.p, n, hi2, lo2);
    RAPID_KERNEL_CHECK();
    return RAPID_OK;
}

// signed (hi, lo) order of NodeIdComparator (:474-500)
__device__ __forceinline__ bool id_less(int64_t ah, int64_t al, int64_t bh, int64_t bl) { return ah < bh || (ah == bh && al < bl); }
// merge of two sorted NodeId lists (a: identifiersSeen, b: the new ones, both strictly increasing): thread i < na places a[i],
// thread na + j places b[j]; an id present in both (or twice in b) sets *dup
__global__ void k_ids_merge(const int64_t* __restrict__ ah, const int64_t* __restrict__ al, int64_t na, const int64_t* __restrict__ bh,
                            const int64_t* __restrict__ bl, int64_t nb, int64_t* __restrict__ oh, int64_t* __restrict__ ol, int32_t* __restrict__ dup) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < na) {
        const int64_t h = ah[t], l = al[t];
        int64_t lo = 0, hi = nb;                             // new ids smaller than a[t]
        while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (id_less(bh[mid], bl[mid], h, l)) lo = mid + 1; else hi = mid; }
        if (lo < nb && bh[lo] == h && bl[lo] == l) atomicCAS(dup, -1, (int32_t)lo);
        oh[t + lo] = h; ol[t + lo] = l;
    } else if (t < na + nb) {
        const int64_t j = t - na;
        const int64_t h = bh[j], l = bl[j];
        int64_t lo = 0, hi = na;                             // seen ids smaller than b[j]
        while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (id_less(ah[mid], al[mid], h, l)) lo = mid + 1; else hi = mid; }
        if (j + 1 < nb && bh[j + 1] == h && bl[j + 1] == l) atomicCAS(dup, -1, (int32_t)j);
        oh[lo + j] = h; ol[lo + j] = l;
    }
}

// merge(identifiersSeen, sorted(add)) into the id scratch, leaving the view alone; RAPID_EUUID_SEEN if a NodeId would be there
// twice.  seen_commit swaps the merged set in: a caller that can still refuse does so in between and the view stays unchanged.
static int32_t seen_merge(View* v, const int64_t* add_hi_dev, const int64_t* add_lo_dev, int64_t n_add) {
    if (n_add <= 0) return RAPID_OK;
    cudaStream_t s = v->stream;
    IdScratch& c = scratch(v)->ids;
    const int64_t tot = v->n_seen + n_add;
    RAPID_CHECK(c.bh.reserve((size_t)n_add)); RAPID_CHECK(c.bl.reserve((size_t)n_add));
    RAPID_CHECK(c.oh.reserve((size_t)tot)); RAPID_CHECK(c.ol.reserve((size_t)tot)); RAPID_CHECK(c.dup.reserve(1));
    RAPID_CHECK(sort_node_ids(v, add_hi_dev, add_lo_dev, n_add, c.bh.p, c.bl.p));
    RAPID_CUDA(cudaMemsetAsync(c.dup.p, 0xff, sizeof(int32_t), s));
    k_ids_merge<<<(unsigned)ceil_div<int64_t>(tot, 256), 256, 0, s>>>(v->seen_hi.p, v->seen_lo.p, v->n_seen, c.bh.p, c.bl.p, n_add, c.oh.p, c.ol.p, c.dup.p);
    RAPID_KERNEL_CHECK();
    int32_t f = -1;
    RAPID_CUDA(cudaMemcpyAsync(&f, c.dup.p, sizeof(f), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    if (f >= 0) { set_error("a NodeId was seen before (UUIDAlreadySeenException)"); return RAPID_EUUID_SEEN; }
    return RAPID_OK;
}
static void seen_commit(View* v, int64_t n_add) {
    if (n_add <= 0) return;
    IdScratch& c = scratch(v)->ids;
    std::swap(v->seen_hi.p, c.oh.p); std::swap(v->seen_hi.cap, c.oh.cap);
    std::swap(v->seen_lo.p, c.ol.p); std::swap(v->seen_lo.cap, c.ol.cap);
    v->n_seen += n_add;
}

template <typename T>
static void swap_buf(DevBuf<T>& a, DevBuf<T>& b) { std::swap(a.p, b.p); std::swap(a.cap, b.cap); }

static int32_t apply_cut_device(View* v, const int32_t* cut_ids, int64_t n_cut, int32_t* out_old_to_new) {
    cudaStream_t s = v->stream;
    const int K = v->K, TB = 256;
    const int64_t n = v->n, tot = v->n + v->nj;
    ViewScratch* sc = scratch(v);
    CutScratch& c = sc->cut;                                  // persistent: no cudaMalloc / cudaFree per view change
    const size_t t1 = (size_t)std::max<int64_t>(tot, 1);
    RAPID_CHECK(c.d_cut.reserve((size_t)std::max<int64_t>(n_cut, 1))); RAPID_CHECK(c.incut.reserve(t1)); RAPID_CHECK(c.newid.reserve(t1 + 1));
    RAPID_CHECK(c.kept.reserve(t1)); RAPID_CHECK(c.len.reserve(t1 + 1)); RAPID_CHECK(c.err.reserve(4)); RAPID_CHECK(c.map.reserve(t1));
    RAPID_CUDA(cudaMemsetAsync(c.incut.p, 0, t1 * sizeof(int32_t), s));
    RAPID_CUDA(cudaMemsetAsync(c.err.p, 0, 4 * sizeof(int32_t), s));       // [0..1] error, [2..3] totals
    if (n_cut) {
        RAPID_CUDA(cudaMemcpyAsync(c.d_cut.p, cut_ids, (size_t)n_cut * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        k_cut_mark<<<(unsigned)ceil_div<int64_t>(n_cut, TB), TB, 0, s>>>(c.d_cut.p, n_cut, n, tot, c.incut.p, c.err.p);
        RAPID_KERNEL_CHECK();
    }
    if (tot) {
        k_cut_keep<<<(unsigned)ceil_div<int64_t>(tot, TB), TB, 0, s>>>(n, tot, c.incut.p, v->host_off.p, c.kept.p, c.len.p);
        RAPID_KERNEL_CHECK();
        RAPID_CUDA(cudaMemcpyAsync(c.newid.p, c.kept.p, (size_t)tot * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
    }
    // kept -> new ids, len -> new byte offsets (exclusive scans; totals on the device)
    RAPID_CHECK(exclusive_scan_i32(c.newid.p, tot, sc->scan_sums, c.err.p + 2, s, nullptr));
    RAPID_CHECK(exclusive_scan_i32(c.len.p, tot, sc->scan_sums, c.err.p + 3, s, nullptr));
    int32_t h[4] = {0, 0, 0, 0}, n_surv = 0;
    RAPID_CUDA(cudaMemcpyAsync(h, c.err.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    if (n < tot) RAPID_CUDA(cudaMemcpyAsync(&n_surv, c.newid.p + n, sizeof(int32_t), cudaMemcpyDeviceToHost, s));   // members that stay = new id of the first joiner
    RAPID_CUDA(cudaStreamSynchronize(s));
    if (h[0] == 1) { set_error("cut id %d outside [0, members + joiners)", h[1]); return RAPID_EINVAL; }
    if (h[0] == 2) {
        set_error("cut names node %d twice", h[1]);
        return h[1] < n ? RAPID_ENOT_IN_RING : RAPID_EALREADY_IN_RING;      // second ringDelete / ringAdd would throw
    }
    const int32_t n2 = h[2], bytes2 = h[3];
    if (n == tot) n_surv = n2;
    const int32_t m = n2 - n_surv;                                          // joiners admitted
    // ---- new endpoint table, keys, NodeIds (built beside the current ones, swapped in at the end) ----------------------------
    const size_t n2s = (size_t)std::max(n2, 1);
    size_t stride2 = 1;
    while (stride2 < n2s) stride2 *= 2;
    RAPID_CHECK(c.hb2.reserve((size_t)std::max(bytes2, 1))); RAPID_CHECK(c.off2.reserve(n2s + 1)); RAPID_CHECK(c.port2.reserve(n2s));
    RAPID_CHECK(c.key2.reserve(stride2 * (size_t)K)); RAPID_CHECK(c.ring2.reserve(n2s * (size_t)K)); RAPID_CHECK(c.sk2.reserve(n2s * (size_t)K));
    if (v->has_node_ids) { RAPID_CHECK(c.nhi2.reserve(n2s)); RAPID_CHECK(c.nlo2.reserve(n2s)); }
    k_cut_endpoints<<<(unsigned)ceil_div<int64_t>(std::max<int64_t>(tot, 1), TB), TB, 0, s>>>(
        tot, c.kept.p, c.newid.p, c.len.p, v->host_off.p, v->host_bytes.p, v->port.p, c.hb2.p, c.off2.p, c.port2.p,
        v->has_node_ids ? v->node_hi.p : nullptr, v->has_node_ids ? v->node_lo.p : nullptr, c.nhi2.p, c.nlo2.p, c.map.p, bytes2, n2);
    RAPID_KERNEL_CHECK();
    if (tot) {
        k_cut_keys<<<(unsigned)ceil_div<int64_t>((int64_t)K * tot, TB), TB, 0, s>>>(K, tot, v->key_stride, stride2, c.kept.p, c.newid.p, v->key.p, c.key2.p);
        RAPID_KERNEL_CHECK();
    }
    // ---- UUID rule for the joiners that come in (:126-128): merged beside identifiersSeen, committed at the swap-in --------------
    const int64_t n_seen_add = v->has_node_ids ? m : 0;
    if (n_seen_add > 0) {
        // the joiners' NodeIds are the last m entries of the new NodeId arrays (joiners follow the surviving members)
        const int32_t rc = seen_merge(v, c.nhi2.p + n_surv, c.nlo2.p + n_surv, n_seen_add);
        if (rc != RAPID_OK) return rc;                                       // UUIDAlreadySeenException: the view is unchanged
    }
    // ---- rings: all K at once ------------------------------------------------------------------------------------------------------
    RAPID_CHECK(c.collision.reserve(3));
    RAPID_CUDA(cudaMemsetAsync(c.collision.p, 0xff, 3 * sizeof(int32_t), s));
    const size_t kn = (size_t)K * (size_t)std::max<int64_t>(n, 1), km = (size_t)K * (size_t)std::max(m, 1);
    RAPID_CHECK(c.flag.reserve(kn)); RAPID_CHECK(c.pos.reserve(kn));
    RAPID_CHECK(c.jk.reserve(km)); RAPID_CHECK(c.jk2.reserve(km)); RAPID_CHECK(c.jv.reserve(km)); RAPID_CHECK(c.jv2.reserve(km));
    if (n > 0) {
        k_cut_ring_flags<<<(unsigned)ceil_div<int64_t>((int64_t)K * n, TB), TB, 0, s>>>(K, n, v->ring.p, c.kept.p, c.flag.p);
        RAPID_KERNEL_CHECK();
        RAPID_CHECK(exclusive_scan_i32_to(c.flag.p, c.pos.p, (int64_t)K * n, sc->scan_sums, s));
    }
    if (m > 0) {
        k_cut_joiner_keys<<<dim3((unsigned)ceil_div<int64_t>(tot - n, TB), (unsigned)K), TB, 0, s>>>(K, n, tot, v->key_stride, c.kept.p, c.newid.p, n_surv, m,
                                                                                                    v->key.p, c.jk.p, c.jv.p);
        RAPID_KERNEL_CHECK();
        if (m <= 32768) {
            k_cut_joiner_rank<<<dim3((unsigned)ceil_div<int32_t>(m, 256), (unsigned)K), 256, 0, s>>>(m, c.jk.p, c.jv.p, c.jk2.p, c.jv2.p, c.collision.p);
            RAPID_KERNEL_CHECK();
        } else {
            for (int k = 0; k < K; ++k)
                RAPID_CHECK(sort_pairs(v, c.jk.p + (size_t)k * m, c.jk2.p + (size_t)k * m, c.jv.p + (size_t)k * m, c.jv2.p + (size_t)k * m, m, s));
            k_cut_joiner_adjacent<<<(unsigned)ceil_div<int64_t>((int64_t)K * m, TB), TB, 0, s>>>(K, m, c.jk2.p, c.jv2.p, c.collision.p);
            RAPID_KERNEL_CHECK();
        }
    }
    if (n + m > 0) {
        k_cut_merge<<<dim3((unsigned)ceil_div<int64_t>(n + m, TB), (unsigned)K), TB, 0, s>>>(n, n_surv, m, v->ring.p, v->sorted_key.p, c.flag.p, c.pos.p, c.newid.p,
                                                                                            c.jk2.p, c.jv2.p, c.ring2.p, c.sk2.p, c.collision.p);
        RAPID_KERNEL_CHECK();
    }
    int32_t coll[3] = {-1, -1, -1};
    RAPID_CUDA(cudaMemcpyAsync(coll, c.collision.p, sizeof(coll), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    if (coll[0] >= 0) {                                                      // the pair's ids index the new endpoint table
        if (same_endpoint(c.hb2.p, c.off2.p, c.port2.p, coll[1], coll[2])) {
            set_error("the cut adds one endpoint twice (new ids %d and %d): NodeAlreadyInRingException", coll[1], coll[2]);
            return RAPID_EALREADY_IN_RING;
        }
        set_error("ring-%d key collision between new ids %d and %d while adding joiners (TreeSet would silently drop one)",
                  coll[0], coll[1], coll[2]);
        return RAPID_EHASH_COLLISION;
    }
    if (out_old_to_new && tot) RAPID_CUDA(cudaMemcpy(out_old_to_new, c.map.p, (size_t)tot * sizeof(int32_t), cudaMemcpyDeviceToHost));
    // ---- swap in: nothing can refuse the cut past this point ----------------------------------------------------------------------
    seen_commit(v, n_seen_add);
    swap_buf(v->host_bytes, c.hb2); swap_buf(v->host_off, c.off2); swap_buf(v->port, c.port2);
    swap_buf(v->key, c.key2); swap_buf(v->ring, c.ring2); swap_buf(v->sorted_key, c.sk2);
    if (v->has_node_ids) { swap_buf(v->node_hi, c.nhi2); swap_buf(v->node_lo, c.nlo2); }
    v->key_stride = stride2;
    v->host_bytes_len = (size_t)bytes2;
    v->n = n2; v->nj = 0;
    ++v->epoch; ++v->member_epoch;
    RAPID_CHECK(v->obs.reserve(stride2 * (size_t)K));
    RAPID_CHECK(v->subj.reserve(n2s * (size_t)K));
    RAPID_CHECK(v->pos0.reserve(n2s));
    if (n2 > 0) {
        k_tables<<<(unsigned)ceil_div<int64_t>((int64_t)n2 * K, TB), TB, 0, s>>>(v->ring.p, n2, K, v->obs.p, v->subj.p, v->pos0.p);
        RAPID_KERNEL_CHECK();
    }
    RAPID_CUDA(cudaStreamSynchronize(s));
    return RAPID_OK;
}

}  // namespace rapid

extern "C" {

// decideViewChange (MembershipService.java:385-444): every node of the decided cut that is a member leaves (ringDelete,
// MembershipView.java:167-201), every other one — a registered joiner — is added (ringAdd, :123-160).  The K rings are
// UPDATED on the device (order-preserving compaction + sorted merge of the joiners, no re-hash, no re-sort of the members);
// ids are renumbered densely: surviving members keep their relative order, the admitted joiners follow in id order, joiners
// not in the cut are dropped.  With NodeIds set (rapid_view_set_node_ids) a joiner whose NodeId is already in
// identifiersSeen is refused (UUIDAlreadySeenException :126-128) and nothing changes.
int32_t rapid_view_apply_cut(rapid_view* v, const int32_t* cut_ids, int64_t n_cut, int32_t* out_old_to_new) {
    if (!v || n_cut < 0 || (n_cut && !cut_ids)) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(v->device);
    return apply_cut_device(v, cut_ids, n_cut, out_old_to_new);
}

// NodeIds of the current members (index = node id): seeds identifiersSeen.  RAPID_EUUID_SEEN if two members share one.
int32_t rapid_view_set_node_ids(rapid_view* v, const int64_t* id_high, const int64_t* id_low) {
    if (!v || (v->n && (!id_high || !id_low))) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(v->device);
    const int64_t tot = v->n + v->nj;
    RAPID_CHECK(v->node_hi.reserve((size_t)std::max<int64_t>(tot, 1))); RAPID_CHECK(v->node_lo.reserve((size_t)std::max<int64_t>(tot, 1)));
    RAPID_CUDA(cudaMemsetAsync(v->node_hi.p, 0, (size_t)std::max<int64_t>(tot, 1) * sizeof(int64_t), v->stream));
    RAPID_CUDA(cudaMemsetAsync(v->node_lo.p, 0, (size_t)std::max<int64_t>(tot, 1) * sizeof(int64_t), v->stream));
    if (v->n) {
        RAPID_CUDA(cudaMemcpyAsync(v->node_hi.p, id_high, (size_t)v->n * sizeof(int64_t), cudaMemcpyHostToDevice, v->stream));
        RAPID_CUDA(cudaMemcpyAsync(v->node_lo.p, id_low, (size_t)v->n * sizeof(int64_t), cudaMemcpyHostToDevice, v->stream));
    }
    RAPID_CUDA(cudaStreamSynchronize(v->stream));
    v->n_seen = 0;
    const int32_t rc = seen_merge(v, v->node_hi.p, v->node_lo.p, v->n);
    if (rc != RAPID_OK) return rc;
    seen_commit(v, v->n);
    v->has_node_ids = true;
    return RAPID_OK;
}

// NodeIds of registered joiners [first_joiner_id, first_joiner_id + count) (AlertMessage.nodeId of their UP alerts,
// MembershipService.java:677-685); checked against identifiersSeen when a cut admits them.
int32_t rapid_view_set_joiner_ids(rapid_view* v, int32_t first_joiner_id, int64_t count, const int64_t* id_high, const int64_t* id_low) {
    if (!v || count < 0 || (count && (!id_high || !id_low))) { set_error("bad arguments"); return RAPID_EINVAL; }
    if (!v->has_node_ids) { set_error("rapid_view_set_node_ids first"); return RAPID_EINVAL; }
    if (first_joiner_id < v->n || (int64_t)first_joiner_id + count > v->n + v->nj) { set_error("not registered joiners"); return RAPID_EINVAL; }
    DeviceGuard g(v->device);
    if (count) {
        RAPID_CUDA(cudaMemcpyAsync(v->node_hi.p + first_joiner_id, id_high, (size_t)count * sizeof(int64_t), cudaMemcpyHostToDevice, v->stream));
        RAPID_CUDA(cudaMemcpyAsync(v->node_lo.p + first_joiner_id, id_low, (size_t)count * sizeof(int64_t), cudaMemcpyHostToDevice, v->stream));
        RAPID_CUDA(cudaStreamSynchronize(v->stream));
    }
    return RAPID_OK;
}

int32_t rapid_view_expected_observers(const rapid_view* cv, const uint8_t* host, int32_t len, int32_t port, int32_t* out,
                                      int32_t* out_count) {
    rapid_view* v = const_cast<rapid_view*>(cv);   // uses scratch space past the registered endpoints; logically const
    if (!v || !out || !out_count || len < 0 || (len && !host)) { set_error("bad arguments"); return RAPID_EINVAL; }
    if (v->n == 0) { *out_count = 0; return RAPID_OK; }
    DeviceGuard g(v->device);
    const int64_t first = v->n + v->nj;
    RAPID_CHECK(ensure_total_capacity(v, first + 1));
    const int32_t off[2] = {0, len};
    static const uint8_t dummy = 0;
    size_t added = 0;
    RAPID_CHECK(upload_endpoints(v, 1, len ? host : &dummy, off, &port, &added));
    std::vector<int32_t> flags;
    int32_t rc = joiner_rows(v, first, 1, flags);
    if (rc == RAPID_OK) {
        cudaError_t e = cudaMemcpy(out, v->obs.p + (size_t)first * v->K, (size_t)v->K * sizeof(int32_t), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) rc = cuda_fail(e, "copy", __FILE__, __LINE__);
    }
    pop_endpoints(v, added);
    if (rc == RAPID_OK) *out_count = v->K;
    return rc;
}

static int32_t config_id_from(rapid_view* v, const int64_t* hi_sorted_dev, const int64_t* lo_sorted_dev, int64_t n_ids, int64_t* out) {
    cudaStream_t s = v->stream;
    const int TB = 256;
    DevBuf<unsigned long long> acc;
    RAPID_CHECK(acc.reserve(1));
    RAPID_CUDA(cudaMemsetAsync(acc.p, 0, sizeof(unsigned long long), s));
    const int64_t M = 2 * n_ids + 2 * v->n;
    const int64_t threads = std::max<int64_t>(1, ceil_div<int64_t>(M, 32));
    k_config_id<<<(unsigned)ceil_div<int64_t>(threads, TB), TB, 0, s>>>(hi_sorted_dev, lo_sorted_dev, nullptr, n_ids, v->host_bytes.p, v->host_off.p,
                                                                        v->port.p, v->ring.p, v->n, acc.p);
    RAPID_KERNEL_CHECK();
    unsigned long long h = 0;
    RAPID_CUDA(cudaMemcpyAsync(&h, acc.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    RAPID_CUDA(cudaStreamSynchronize(s));
    *out = (int64_t)h;
    return RAPID_OK;
}

// Configuration.getConfigurationId (:544-556) over caller-supplied identifiers (any order: sorted here by signed (high, low))
int32_t rapid_view_config_id(const rapid_view* cv, const int64_t* id_high, const int64_t* id_low, int64_t n_ids, int64_t* out) {
    rapid_view* v = const_cast<rapid_view*>(cv);
    if (!v || !out || n_ids < 0 || (n_ids && (!id_high || !id_low))) { set_error("bad arguments"); return RAPID_EINVAL; }
    DeviceGuard g(v->device);
    cudaStream_t s = v->stream;
    DevBuf<int64_t> dh, dl, sh, sl;
    const size_t m = (size_t)std::max<int64_t>(1, n_ids);
    RAPID_CHECK(dh.reserve(m)); RAPID_CHECK(dl.reserve(m)); RAPID_CHECK(sh.reserve(m)); RAPID_CHECK(sl.reserve(m));
    if (n_ids) {
        RAPID_CUDA(cudaMemcpyAsync(dh.p, id_high, (size_t)n_ids * sizeof(int64_t), cudaMemcpyHostToDevice, s));
        RAPID_CUDA(cudaMemcpyAsync(dl.p, id_low, (size_t)n_ids * sizeof(int64_t), cudaMemcpyHostToDevice, s));
        RAPID_CHECK(sort_node_ids(v, dh.p, dl.p, n_ids, sh.p, sl.p));       // NodeIdComparator (:474-500): signed (high, low)
    }
    return config_id_from(v, sh.p, sl.p, n_ids, out);
}

// getCurrentConfigurationId (:360-372) from the view's OWN identifiersSeen (rapid_view_set_node_ids; grows with every admitted
// joiner, never shrinks — ids of removed nodes stay, :167-201) and its ring 0: nothing but the 8-byte result leaves the device.
int32_t rapid_view_current_config_id(const rapid_view* cv, int64_t* out) {
    rapid_view* v = const_cast<rapid_view*>(cv);
    if (!v || !out) { set_error("bad arguments"); return RAPID_EINVAL; }
    if (!v->has_node_ids) { set_error("rapid_view_set_node_ids first"); return RAPID_EINVAL; }
    DeviceGuard g(v->device);
    return config_id_from(v, v->seen_hi.p, v->seen_lo.p, v->n_seen, out);
}

}  // extern "C"
