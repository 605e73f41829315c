// Shared internals of librapid_b200.so (sm_90a, H100).  Nothing here is part of the C ABI.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/rapid_b200.h"

namespace rapid {

// ---------------------------------------------------------------- error plumbing
void set_error(const char* fmt, ...);
int32_t cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define RAPID_CUDA(call)                                                                  \
    do {                                                                                  \
        cudaError_t _e = (call);                                                          \
        if (_e != cudaSuccess) return ::rapid::cuda_fail(_e, #call, __FILE__, __LINE__);  \
    } while (0)

#define RAPID_CHECK(expr)                 \
    do {                                  \
        int32_t _rc = (expr);             \
        if (_rc != RAPID_OK) return _rc;  \
    } while (0)

#define RAPID_KERNEL_CHECK() RAPID_CUDA(cudaGetLastError())

// ---------------------------------------------------------------- small helpers
// SMs of the target GPU (H100 SXM: 132).  It only caps grid-stride launches at a few waves and is the fallback if the device
// attribute cannot be read; grids that must be co-resident are sized from the device's own attributes.
constexpr int TARGET_SMS = 132;

template <typename T>
static inline T ceil_div(T a, T b) { return (a + b - 1) / b; }

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// A growable device buffer (plain cudaMalloc; sizes are in elements).
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t cap = 0;
    ~DevBuf() { release(); }
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    // ensure capacity; contents are NOT preserved unless keep == true
    int32_t reserve(size_t n, bool keep = false, cudaStream_t s = 0) {
        if (n <= cap) return RAPID_OK;
        size_t ncap = cap ? cap : 1;
        while (ncap < n) ncap *= 2;
        // scratch buffers: the FIRST allocation is exact (the big state arrays are allocated once), a later one grows
        // geometrically — cudaFree synchronises the device, which an asynchronous stream of batches of slowly growing size
        // would otherwise pay on every batch
        if (!keep && cap == 0) ncap = n;
        T* np = nullptr;
        cudaError_t e = cudaMalloc((void**)&np, ncap * sizeof(T));
        if (e != cudaSuccess) { set_error("cudaMalloc(%zu bytes) failed: %s", ncap * sizeof(T), cudaGetErrorString(e)); cudaGetLastError(); return RAPID_ENOMEM; }
        if (keep && p && cap) {
            e = cudaMemcpyAsync(np, p, cap * sizeof(T), cudaMemcpyDeviceToDevice, s);
            if (e != cudaSuccess) { cudaFree(np); return cuda_fail(e, "grow copy", __FILE__, __LINE__); }
            cudaStreamSynchronize(s);
        }
        if (p) cudaFree(p);
        p = np; cap = ncap;
        return RAPID_OK;
    }
};

// Pinned host staging buffer.
template <typename T>
struct PinnedBuf {
    T* p = nullptr;
    size_t cap = 0;
    ~PinnedBuf() { if (p) cudaFreeHost(p); }
    int32_t reserve(size_t n) {
        if (n <= cap) return RAPID_OK;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        cudaError_t e = cudaMallocHost((void**)&p, n * sizeof(T));
        if (e != cudaSuccess) { set_error("cudaMallocHost failed: %s", cudaGetErrorString(e)); cudaGetLastError(); return RAPID_ENOMEM; }
        cap = n;
        return RAPID_OK;
    }
};

// ---------------------------------------------------------------- hashes (host + device)
#ifdef __CUDACC__
#define RAPID_HD __host__ __device__ __forceinline__
#else
#define RAPID_HD inline
#endif

RAPID_HD uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }

RAPID_HD uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}

// The order of RAPID_DELIVERY_SHUFFLED_BATCHES (include/rapid_b200.h): global receiver g meets the n batches of a sequence as
// batch_order_at(o, 0), batch_order_at(o, 1), ..., a keyed permutation of [0, n) computed in O(1) per step and no memory: a 4-round
// Feistel network on 2w bits (4^w >= n) made a bijection of [0, n) by cycle walking (4^w / n walks expected: < 4 above n = 256).
// w starts at 4: on halves of 1-3 bits a 4-round Feistel network reaches a visibly skewed set of orders (for n = 5, some of the 120
// orders come 8 times as often as others), on 4-bit halves the orders of small n pass a chi-square test of uniformity.
struct BatchOrder { uint64_t key, m; int64_t n; int w; };

RAPID_HD BatchOrder batch_order_init(uint64_t seed, int64_t g, int64_t n) {
    BatchOrder o;
    o.key = splitmix64(seed + (uint64_t)g);
    o.n = n;
    o.w = 4;
    while (((int64_t)1 << (2 * o.w)) < n) ++o.w;
    o.m = ((uint64_t)1 << o.w) - 1;
    return o;
}

RAPID_HD uint64_t batch_order_feistel(const BatchOrder& o, uint64_t v) {
    uint64_t a = v >> o.w, b = v & o.m;
    for (int i = 0; i < 4; ++i) {
        const uint64_t t = a ^ (splitmix64(o.key ^ ((uint64_t)(i + 1) << 58) ^ b) & o.m);
        a = b;
        b = t;
    }
    return (a << o.w) | b;
}

RAPID_HD int64_t batch_order_at(const BatchOrder& o, int64_t j) {
    if (o.n <= 1) return j;
    uint64_t v = batch_order_feistel(o, (uint64_t)j);
    while (v >= (uint64_t)o.n) v = batch_order_feistel(o, v);
    return (int64_t)v;
}

// Per-element mixers of the order-independent proposal fingerprint (rapid_proposal_fingerprint).
RAPID_HD uint64_t fp_mix1(int32_t id) { return splitmix64((uint64_t)(uint32_t)id ^ 0x52415049445F4831ULL); }
RAPID_HD uint64_t fp_mix2(int32_t id) { return splitmix64(((uint64_t)(uint32_t)id * 0xD6E8FEB86659FD93ULL) ^ 0x52415049445F4832ULL); }

#ifdef __CUDACC__
// Open addressing over proposal fingerprints (a, b, l) = (h1, h2, len) in a table of T (a power of two) slots, empty slots -1:
// item s claims the slot of its fingerprint, and the slot keeps the LOWEST item holding it (atomicCAS, then atomicMin).
// fp(i, &a, &b, &l) reads item i's fingerprint.  Returns the slot.  The proposal grouping (group_proposals, cd_census.cu) numbers
// the census's classes and the wire encoder's bodies this way.
template <typename FP>
__device__ __forceinline__ uint32_t fp_table_claim(int32_t* table, uint32_t T, int32_t s, uint64_t a, uint64_t b, int32_t l, const FP& fp) {
    uint32_t pos = (uint32_t)(splitmix64(a ^ (b * 0x9E3779B97F4A7C15ULL) ^ (uint64_t)l) >> 32) & (T - 1);
    for (;;) {
        int32_t cur = table[pos];
        if (cur < 0) {
            cur = atomicCAS(&table[pos], -1, s);
            if (cur < 0) return pos;
        }
        uint64_t ca, cb; int32_t cl;
        fp(cur, &ca, &cb, &cl);
        if (ca == a && cb == b && cl == l) { atomicMin(&table[pos], s); return pos; }
        pos = (pos + 1) & (T - 1);
    }
}
#endif

#define XXP1 0x9E3779B185EBCA87ULL
#define XXP2 0xC2B2AE3D27D4EB4FULL
#define XXP3 0x165667B19E3779F9ULL
#define XXP4 0x85EBCA77C2B2AE63ULL
#define XXP5 0x27D4EB2F165667C5ULL

RAPID_HD uint64_t xx_round(uint64_t acc, uint64_t in) { acc += in * XXP2; acc = rotl64(acc, 31); return acc * XXP1; }
RAPID_HD uint64_t xx_merge(uint64_t acc, uint64_t v) { v = xx_round(0, v); acc ^= v; return acc * XXP1 + XXP4; }
RAPID_HD uint64_t xx_avalanche(uint64_t h) { h ^= h >> 33; h *= XXP2; h ^= h >> 29; h *= XXP3; h ^= h >> 32; return h; }

RAPID_HD uint64_t xx_read64(const uint8_t* p) { uint64_t v = 0; for (int i = 7; i >= 0; --i) v = (v << 8) | p[i]; return v; }
RAPID_HD uint32_t xx_read32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

// XXH64 of a byte string (LongHashFunction.xx(seed).hashBytes)
RAPID_HD uint64_t xxh64_bytes(const uint8_t* p, int len, uint64_t seed) {
    const uint8_t* const end = p + len;
    uint64_t h;
    if (len >= 32) {
        const uint8_t* const limit = end - 32;
        uint64_t v1 = seed + XXP1 + XXP2, v2 = seed + XXP2, v3 = seed, v4 = seed - XXP1;
        do {
            v1 = xx_round(v1, xx_read64(p)); p += 8;
            v2 = xx_round(v2, xx_read64(p)); p += 8;
            v3 = xx_round(v3, xx_read64(p)); p += 8;
            v4 = xx_round(v4, xx_read64(p)); p += 8;
        } while (p <= limit);
        h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
        h = xx_merge(h, v1); h = xx_merge(h, v2); h = xx_merge(h, v3); h = xx_merge(h, v4);
    } else {
        h = seed + XXP5;
    }
    h += (uint64_t)len;
    while (p + 8 <= end) { h ^= xx_round(0, xx_read64(p)); h = rotl64(h, 27) * XXP1 + XXP4; p += 8; }
    if (p + 4 <= end) { h ^= (uint64_t)xx_read32(p) * XXP1; h = rotl64(h, 23) * XXP2 + XXP3; p += 4; }
    while (p < end) { h ^= (uint64_t)(*p) * XXP5; h = rotl64(h, 11) * XXP1; ++p; }
    return xx_avalanche(h);
}
// LongHashFunction.xx(seed).hashInt(v) == XXH64 of the 4 LE bytes
RAPID_HD uint64_t xxh64_int(int32_t v, uint64_t seed) {
    uint64_t h = seed + XXP5 + 4;
    h ^= (uint64_t)(uint32_t)v * XXP1;
    h = rotl64(h, 23) * XXP2 + XXP3;
    return xx_avalanche(h);
}
// LongHashFunction.xx(seed).hashLong(v) == XXH64 of the 8 LE bytes
RAPID_HD uint64_t xxh64_long(int64_t v, uint64_t seed) {
    uint64_t h = seed + XXP5 + 8;
    h ^= xx_round(0, (uint64_t)v);
    h = rotl64(h, 27) * XXP1 + XXP4;
    return xx_avalanche(h);
}
// AddressComparator.computeHash (MembershipView.java:579-582)
RAPID_HD int64_t ring_key(const uint8_t* host, int len, int32_t port, int k) {
    return (int64_t)(xxh64_bytes(host, len, (uint64_t)k) * 31ULL + xxh64_int(port, (uint64_t)k));
}

// ---------------------------------------------------------------- handle layouts shared between files
struct View {
    int device = 0;
    int K = 0;
    int64_t n = 0;          // members
    int64_t nj = 0;         // registered joiners (ids n .. n+nj-1)
    uint64_t epoch = 1;     // bumped whenever the endpoint -> id dictionary changes (joiners registered, cut applied)
    uint64_t member_epoch = 1;   // bumped only when the MEMBERS change (a cut was applied): what per-member state hangs off
    cudaStream_t stream = nullptr;
    // endpoints (members then joiners)
    DevBuf<uint8_t> host_bytes;   size_t host_bytes_len = 0;
    DevBuf<int32_t> host_off;     // [n+nj+1]
    DevBuf<int32_t> port;         // [n+nj]
    // NodeIds (MembershipView.java:58-60 identifiersSeen, :126-128 UUIDAlreadySeenException) — optional (rapid_view_set_node_ids)
    bool has_node_ids = false;
    DevBuf<int64_t> node_hi, node_lo;     // [n+nj] NodeId of every endpoint id
    DevBuf<int64_t> seen_hi, seen_lo;     // [n_seen] identifiersSeen, sorted by signed (high, low); only ever grows
    int64_t n_seen = 0;
    void* scratch = nullptr;              // view.cu's sort / scan scratch
    // rings
    DevBuf<int64_t> key;          // [K][ntot_cap]  key of node id on ring k (members + joiners)
    size_t key_stride = 0;        // ntot capacity (row stride of key)
    DevBuf<int64_t> sorted_key;   // [K][n] keys in ring order
    DevBuf<int32_t> ring;         // [K][n] node id at each ring position
    DevBuf<int32_t> pos0;         // [n] ring-0 position of member id
    DevBuf<int32_t> obs;          // [ntot_cap][K] members: ring successors; joiners: expected observers (predecessors)
    DevBuf<int32_t> subj;         // [n][K]        ring predecessors
};

}  // namespace rapid

// the opaque ABI handle types are thin tags over the internal structs
struct rapid_view : rapid::View {};
