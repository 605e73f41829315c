// Expansion of the K-ring monitoring overlay: the extreme eigenvalues of a view's observer graph below the trivial one.
//
// The graph: A = sum_k (P_k + P_k^T), P_k = "successor on ring k", i.e. A[v][obs[v][k]] += 1 and A[v][subj[v][k]] += 1 for every k,
// multiplicities kept (a node that observes another on m rings contributes m).  A is symmetric, every row sums to 2K, the top
// eigenvalue is 2K with the all-ones vector.  rapid_view_overlay_spectrum reports the largest (lambda2) and the smallest
// (lambda_min) eigenvalue of A restricted to the complement of the all-ones vector; max(|lambda2|, |lambda_min|) / 2K is the figure
// the Rapid paper quotes (< 0.45 at K = 10).  Registered joiners are not part of the graph.
//
// Method: Lanczos in the complement of the all-ones vector, fp64, the basis kept in HBM and every new vector re-orthogonalised
// against all of it (one classical Gram-Schmidt pass after the three-term recurrence): the spectrum below 2K is the edge of a dense
// bulk, plain Lanczos would lose orthogonality long before the edge converges.  One step j is
//   k_overlay_apply     v_j = s * t (the normalised basis vector, stored), y = A v_j, block partials of alpha_j = y.v_j and sum(y)
//   k_overlay_alpha     the partials combined in a fixed order -> alpha_j, mean(y)
//   k_overlay_project   y -= mean + alpha_j v_j + beta_{j-1} v_{j-1}; block partials of the dots V_i.y, one warp per basis vector
//   k_overlay_coeffs    the partials combined in a fixed order -> c_i
//   k_overlay_subtract  y -= sum_i c_i v_i; block partials of |y|^2
//   k_overlay_norm      the partials combined in a fixed order -> beta_j = |y|, s = 1 / beta_j; y becomes the next t
// Every sum over nodes is per-block partials combined by one small block in a fixed order (no floating-point atomics), so two calls
// with the same seed on the same view return the same bits.  The start vector is t[v] = 2 u - 1, u = (splitmix64(seed + v) >> 11)
// * 2^-53, mean removed, normalised.  The m x m tridiagonal eigenproblem is solved on the host (implicit QL, carrying the last row
// of the eigenvector matrix) from the alpha and beta read back every few steps; the residual of a Ritz value theta_i is
// |beta_m * s_mi|, a bound on the distance from theta_i to an eigenvalue of A.
#include <float.h>
#include <math.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace rapid {

constexpr int OV_TB = 256;                       // threads of every block here
constexpr int OV_MAX_BLOCKS = 8 * TARGET_SMS;    // grid-stride kernels: at most this many per-block partials to combine
constexpr int OV_PROJECT_BLOCKS = 4 * TARGET_SMS;
enum { OV_MEAN = 0, OV_ALPHA = 1, OV_BETA_PREV = 2, OV_SCALE = 3, OV_SCALARS = 4 };   // scal[]: the step's scalars on the device

// sum over the block, the same order every time: warp shuffles, then warp 0 over the warp sums.  Valid in thread 0.
__device__ __forceinline__ double block_sum(double v) {
    __shared__ double sm[OV_TB / 32];
    __syncthreads();                              // sm may still be read from the previous call
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
        v = threadIdx.x < OV_TB / 32 ? sm[threadIdx.x] : 0.0;
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    }
    return v;
}
// sum of p[0..nb) by one block (thread t takes t, t + 256, ... in order)
__device__ __forceinline__ double combine(const double* __restrict__ p, int nb) {
    double v = 0.0;
    for (int b = threadIdx.x; b < nb; b += OV_TB) v += p[b];
    return block_sum(v);
}

__global__ void __launch_bounds__(OV_TB) k_overlay_start(double* __restrict__ t, int64_t n, uint64_t seed, double* __restrict__ part) {
    double acc = 0.0;
    for (int64_t v = (int64_t)blockIdx.x * OV_TB + threadIdx.x; v < n; v += (int64_t)gridDim.x * OV_TB) {
        const double x = 2.0 * ((double)(splitmix64(seed + (uint64_t)v) >> 11) * 0x1.0p-53) - 1.0;
        t[v] = x;
        acc += x;
    }
    acc = block_sum(acc);
    if (threadIdx.x == 0) part[blockIdx.x] = acc;
}
__global__ void __launch_bounds__(OV_TB) k_overlay_mean(const double* __restrict__ part, int nb, int64_t n, double* __restrict__ scal) {
    const double s = combine(part, nb);
    if (threadIdx.x == 0) scal[OV_MEAN] = s / (double)n;
}
__global__ void __launch_bounds__(OV_TB) k_overlay_centre(double* __restrict__ t, int64_t n, const double* __restrict__ scal,
                                                          double* __restrict__ part) {
    const double mean = scal[OV_MEAN];
    double acc = 0.0;
    for (int64_t v = (int64_t)blockIdx.x * OV_TB + threadIdx.x; v < n; v += (int64_t)gridDim.x * OV_TB) {
        const double x = t[v] - mean;
        t[v] = x;
        acc += x * x;
    }
    acc = block_sum(acc);
    if (threadIdx.x == 0) part[blockIdx.x] = acc;
}
// |y| from the partials of |y|^2: beta[step] (step 0 = the start vector, not a beta), the scale of the next basis vector, and the
// beta the next step's recurrence subtracts.  A vector that is rounding noise (the Krylov space is exhausted) gets scale 0.
__global__ void __launch_bounds__(OV_TB) k_overlay_norm(const double* __restrict__ part, int nb, int step, double tiny,
                                                        double* __restrict__ scal, double* __restrict__ beta) {
    const double s = combine(part, nb);
    if (threadIdx.x == 0) {
        const double nrm = sqrt(s);
        if (step > 0) beta[step - 1] = nrm;
        scal[OV_BETA_PREV] = step > 0 ? nrm : 0.0;
        scal[OV_SCALE] = nrm > tiny ? 1.0 / nrm : 0.0;
    }
}

// sum of x over one W-int piece of a table row
template <int W> struct RowPiece;
template <> struct RowPiece<1> { typedef int32_t T; static __device__ __forceinline__ double sum(T r, const double* __restrict__ x) { return __ldg(x + r); } };
template <> struct RowPiece<2> { typedef int2 T; static __device__ __forceinline__ double sum(T r, const double* __restrict__ x) { return __ldg(x + r.x) + __ldg(x + r.y); } };
template <> struct RowPiece<4> { typedef int4 T; static __device__ __forceinline__ double sum(T r, const double* __restrict__ x) { return (__ldg(x + r.x) + __ldg(x + r.y)) + (__ldg(x + r.z) + __ldg(x + r.w)); } };

// The operator, one thread per node: y[v] = s * sum_k t[obs[v][k]] + t[subj[v][k]], the node-major 4K-byte rows of both tables read
// as K / W loads of W ints (W = 4 when K % 4 == 0, 2 when K is even: a K = 10 row is 40 B, five 64-bit loads), t gathered through the
// read-only path.  In the same pass: the normalised basis vector vj[v] = s * t[v] is stored, and the block's share of alpha = y.vj and
// of sum(y) go to part[block] and part[gridDim.x + block].
template <int W>
__global__ void __launch_bounds__(OV_TB) k_overlay_apply(const int32_t* __restrict__ obs, const int32_t* __restrict__ subj, int K, int64_t n,
                                                         const double* __restrict__ t, const double* __restrict__ scal,
                                                         double* __restrict__ vj, double* __restrict__ y, double* __restrict__ part) {
    typedef typename RowPiece<W>::T Piece;
    const double s = scal[OV_SCALE];
    const int pieces = K / W;
    double a_alpha = 0.0, a_sum = 0.0;
    for (int64_t v = (int64_t)blockIdx.x * OV_TB + threadIdx.x; v < n; v += (int64_t)gridDim.x * OV_TB) {
        const Piece* ro = reinterpret_cast<const Piece*>(obs + (size_t)v * K);
        const Piece* rs = reinterpret_cast<const Piece*>(subj + (size_t)v * K);
        double acc = 0.0;
        for (int c = 0; c < pieces; ++c) acc += RowPiece<W>::sum(ro[c], t) + RowPiece<W>::sum(rs[c], t);
        const double yv = s * acc, xv = s * t[v];
        vj[v] = xv;
        y[v] = yv;
        a_alpha += yv * xv;
        a_sum += yv;
    }
    a_alpha = block_sum(a_alpha);
    a_sum = block_sum(a_sum);
    if (threadIdx.x == 0) { part[blockIdx.x] = a_alpha; part[gridDim.x + blockIdx.x] = a_sum; }
}
__global__ void __launch_bounds__(OV_TB) k_overlay_alpha(const double* __restrict__ part, int nb, int64_t n, int step,
                                                         double* __restrict__ scal, double* __restrict__ alpha) {
    const double a = combine(part, nb);
    const double s = combine(part + nb, nb);
    if (threadIdx.x == 0) { scal[OV_ALPHA] = a; alpha[step - 1] = a; scal[OV_MEAN] = s / (double)n; }
}

// Block b owns the nodes [b * chunk, (b + 1) * chunk).  First the three-term recurrence and the all-ones direction on its nodes,
// y -= mean + alpha v_j + beta_{j-1} v_{j-1}; then warp w takes the basis vectors i = w, w + 8, ... < j and leaves the block's share
// of v_i . y in pd[b * j + i]: each lane sums its nodes in order, the lanes are combined by shuffles.  The basis streams from HBM once;
// the block's piece of y is re-read from cache.
__global__ void __launch_bounds__(OV_TB) k_overlay_project(const double* __restrict__ basis, int64_t n, int j, int64_t chunk,
                                                           const double* __restrict__ scal, double* __restrict__ y, double* __restrict__ pd) {
    const int64_t lo = (int64_t)blockIdx.x * chunk, hi = min(n, lo + chunk);
    const double mean = scal[OV_MEAN], alpha = scal[OV_ALPHA], beta = scal[OV_BETA_PREV];
    const double* vj = basis + (size_t)(j - 1) * n;
    const double* vp = basis + (size_t)(j > 1 ? j - 2 : 0) * n;
    for (int64_t v = lo + threadIdx.x; v < hi; v += OV_TB) {
        double r = y[v] - mean - alpha * vj[v];
        if (j > 1) r -= beta * vp[v];
        y[v] = r;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (int i = threadIdx.x >> 5; i < j; i += OV_TB / 32) {
        const double* vi = basis + (size_t)i * n;
        double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
        int64_t v = lo + lane;
        for (; v + 96 < hi; v += 128) {
            a0 += vi[v] * y[v];
            a1 += vi[v + 32] * y[v + 32];
            a2 += vi[v + 64] * y[v + 64];
            a3 += vi[v + 96] * y[v + 96];
        }
        for (; v < hi; v += 32) a0 += vi[v] * y[v];
        double a = (a0 + a1) + (a2 + a3);
        for (int o = 16; o > 0; o >>= 1) a += __shfl_down_sync(0xffffffffu, a, o);
        if (lane == 0) pd[(size_t)blockIdx.x * j + i] = a;
    }
}
__global__ void __launch_bounds__(OV_TB) k_overlay_coeffs(const double* __restrict__ pd, int nb, int j, double* __restrict__ c) {
    const int i = blockIdx.x * OV_TB + threadIdx.x;
    if (i >= j) return;
    double a = 0.0;
    for (int b = 0; b < nb; ++b) a += pd[(size_t)b * j + i];
    c[i] = a;
}
// y -= sum_i c_i v_i (i ascending), one thread per node; the block's share of |y|^2 to part[block]
__global__ void __launch_bounds__(OV_TB) k_overlay_subtract(const double* __restrict__ basis, int64_t n, int j, const double* __restrict__ c,
                                                            double* __restrict__ y, double* __restrict__ part) {
    __shared__ double sc[RAPID_OVERLAY_MAX_STEPS];
    for (int i = threadIdx.x; i < j; i += OV_TB) sc[i] = c[i];
    __syncthreads();
    double acc = 0.0;
    for (int64_t v = (int64_t)blockIdx.x * OV_TB + threadIdx.x; v < n; v += (int64_t)gridDim.x * OV_TB) {
        double r = y[v];
        const double* col = basis + v;
        int i = 0;
        for (; i + 4 <= j; i += 4) {
            const double b0 = col[(size_t)i * n], b1 = col[(size_t)(i + 1) * n], b2 = col[(size_t)(i + 2) * n], b3 = col[(size_t)(i + 3) * n];
            r -= sc[i] * b0;
            r -= sc[i + 1] * b1;
            r -= sc[i + 2] * b2;
            r -= sc[i + 3] * b3;
        }
        for (; i < j; ++i) r -= sc[i] * col[(size_t)i * n];
        y[v] = r;
        acc += r * r;
    }
    acc = block_sum(acc);
    if (threadIdx.x == 0) part[blockIdx.x] = acc;
}

// ------------------------------------------------------------------ host: the tridiagonal eigenproblem
// Implicit QL on the symmetric tridiagonal (d[0..m), e[0..m-1) off the diagonal): d becomes the eigenvalues, z[i] the LAST component
// of eigenvector i (z starts as the last row of the identity and takes every rotation).  false if a value does not converge.
static bool tridiagonal_ql(std::vector<double>& d, std::vector<double>& e, std::vector<double>& z) {
    const int m = (int)d.size();
    e.resize((size_t)m);
    e[(size_t)m - 1] = 0.0;
    z.assign((size_t)m, 0.0);
    z[(size_t)m - 1] = 1.0;
    for (int l = 0; l < m; ++l) {
        for (int iter = 0;; ++iter) {
            int q = l;
            for (; q < m - 1; ++q)
                if (fabs(e[q]) <= DBL_EPSILON * (fabs(d[q]) + fabs(d[q + 1])) + DBL_MIN) break;
            if (q == l) break;
            if (iter == 60) return false;
            double g = (d[l + 1] - d[l]) / (2.0 * e[l]);
            double r = hypot(g, 1.0);
            g = d[q] - d[l] + e[l] / (g + copysign(r, g));
            double s = 1.0, c = 1.0, p = 0.0;
            int i = q - 1;
            for (; i >= l; --i) {
                double f = s * e[i];
                const double b = c * e[i];
                r = hypot(f, g);
                e[i + 1] = r;
                if (r == 0.0) { d[i + 1] -= p; e[q] = 0.0; break; }
                s = f / r;
                c = g / r;
                g = d[i + 1] - p;
                r = (d[i] - g) * s + 2.0 * c * b;
                p = s * r;
                d[i + 1] = g + p;
                g = c * r - b;
                f = z[i + 1];
                z[i + 1] = s * z[i] + c * f;
                z[i] = c * z[i] - s * f;
            }
            if (r == 0.0 && i >= l) continue;
            d[l] -= p;
            e[l] = g;
            e[q] = 0.0;
        }
    }
    return true;
}

struct Ritz { double hi, lo, residual; };
// the two ends of the spectrum of T_m = tridiag(beta, alpha, beta) and the larger of their residuals |beta_m * z|
static bool ritz_ends(const double* alpha, const double* beta, int m, Ritz* out) {
    std::vector<double> d(alpha, alpha + m), e(beta, beta + m - 1), z;
    if (!tridiagonal_ql(d, e, z)) return false;
    const int ih = (int)(std::max_element(d.begin(), d.end()) - d.begin());
    const int il = (int)(std::min_element(d.begin(), d.end()) - d.begin());
    out->hi = d[(size_t)ih];
    out->lo = d[(size_t)il];
    out->residual = fabs(beta[m - 1]) * std::max(fabs(z[(size_t)ih]), fabs(z[(size_t)il]));
    return true;
}

struct OverlayScratch {                           // of one call: allocated once before the first step, freed when the call returns
    DevBuf<double> basis, t, y, part, pd, c, alpha, beta, scal;
};

template <int W>
static void launch_apply(const View* v, int nb, const double* t, const double* scal, double* vj, double* y, double* part, cudaStream_t s) {
    k_overlay_apply<W><<<nb, OV_TB, 0, s>>>(v->obs.p, v->subj.p, v->K, v->n, t, scal, vj, y, part);
}

static int32_t overlay_spectrum(const View* v, uint64_t seed, double tol, int32_t max_steps, Ritz* out, int32_t* out_steps, float* out_ms) {
    cudaStream_t s = v->stream;
    const int64_t n = v->n;
    const int K = v->K;
    const int m_max = (int)std::min<int64_t>(max_steps, n - 1);          // the complement of the all-ones vector has n - 1 dimensions
    const int nb = (int)std::min<int64_t>(ceil_div<int64_t>(n, OV_TB), OV_MAX_BLOCKS);
    const int64_t chunk = std::max<int64_t>(ceil_div<int64_t>(n, OV_PROJECT_BLOCKS), 128);
    const int nbp = (int)ceil_div<int64_t>(n, chunk);
    const double scale = 2.0 * K, tiny = 1e-12 * scale;

    OverlayScratch sc;
    RAPID_CHECK(sc.basis.reserve((size_t)m_max * (size_t)n));
    RAPID_CHECK(sc.t.reserve((size_t)n)); RAPID_CHECK(sc.y.reserve((size_t)n));
    RAPID_CHECK(sc.part.reserve(2 * (size_t)nb)); RAPID_CHECK(sc.pd.reserve((size_t)nbp * (size_t)m_max)); RAPID_CHECK(sc.c.reserve((size_t)m_max));
    RAPID_CHECK(sc.alpha.reserve((size_t)m_max)); RAPID_CHECK(sc.beta.reserve((size_t)m_max)); RAPID_CHECK(sc.scal.reserve(OV_SCALARS));
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    RAPID_CUDA(cudaEventCreate(&e0));
    if (cudaEventCreate(&e1) != cudaSuccess) { cudaEventDestroy(e0); return cuda_fail(cudaGetLastError(), "event", __FILE__, __LINE__); }
    struct Events { cudaEvent_t a, b; ~Events() { cudaEventDestroy(a); cudaEventDestroy(b); } } events{e0, e1};

    RAPID_CUDA(cudaEventRecord(e0, s));
    k_overlay_start<<<nb, OV_TB, 0, s>>>(sc.t.p, n, seed, sc.part.p);
    k_overlay_mean<<<1, OV_TB, 0, s>>>(sc.part.p, nb, n, sc.scal.p);
    k_overlay_centre<<<nb, OV_TB, 0, s>>>(sc.t.p, n, sc.scal.p, sc.part.p);
    k_overlay_norm<<<1, OV_TB, 0, s>>>(sc.part.p, nb, 0, 0.0, sc.scal.p, sc.beta.p);
    RAPID_KERNEL_CHECK();

    std::vector<double> alpha((size_t)m_max), beta((size_t)m_max);
    double *t = sc.t.p, *y = sc.y.p;
    int m = 0;                                                            // steps whose alpha and beta the host has judged
    bool done = false;
    for (int j = 1; j <= m_max && !done; ++j) {
        double* vj = sc.basis.p + (size_t)(j - 1) * n;
        if (K % 4 == 0) launch_apply<4>(v, nb, t, sc.scal.p, vj, y, sc.part.p, s);
        else if (K % 2 == 0) launch_apply<2>(v, nb, t, sc.scal.p, vj, y, sc.part.p, s);
        else launch_apply<1>(v, nb, t, sc.scal.p, vj, y, sc.part.p, s);
        k_overlay_alpha<<<1, OV_TB, 0, s>>>(sc.part.p, nb, n, j, sc.scal.p, sc.alpha.p);
        k_overlay_project<<<nbp, OV_TB, 0, s>>>(sc.basis.p, n, j, chunk, sc.scal.p, y, sc.pd.p);
        k_overlay_coeffs<<<ceil_div(j, OV_TB), OV_TB, 0, s>>>(sc.pd.p, nbp, j, sc.c.p);
        k_overlay_subtract<<<nb, OV_TB, 0, s>>>(sc.basis.p, n, j, sc.c.p, y, sc.part.p);
        k_overlay_norm<<<1, OV_TB, 0, s>>>(sc.part.p, nb, j, tiny, sc.scal.p, sc.beta.p);
        RAPID_KERNEL_CHECK();
        std::swap(t, y);
        // the host looks at every step while the problem is tiny, then every 8th: a look drains the stream
        if (j > 16 && j % 8 != 0 && j != m_max) continue;
        RAPID_CUDA(cudaMemcpyAsync(alpha.data() + m, sc.alpha.p + m, (size_t)(j - m) * sizeof(double), cudaMemcpyDeviceToHost, s));
        RAPID_CUDA(cudaMemcpyAsync(beta.data() + m, sc.beta.p + m, (size_t)(j - m) * sizeof(double), cudaMemcpyDeviceToHost, s));
        RAPID_CUDA(cudaStreamSynchronize(s));
        int use = j;                                                      // beta_i ~ 0: the Krylov space ended at step i, T_i is exact
        for (int i = m; i < j; ++i)
            if (beta[(size_t)i] <= tiny) { use = i + 1; break; }
        m = j;
        if (!ritz_ends(alpha.data(), beta.data(), use, out)) { set_error("overlay spectrum: the tridiagonal QL iteration did not converge (step %d)", j); return RAPID_ECUDA; }
        done = use < j || out->residual <= tol * scale;
    }
    RAPID_CUDA(cudaEventRecord(e1, s));
    RAPID_CUDA(cudaEventSynchronize(e1));
    float ms = 0.f;
    RAPID_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    *out_steps = m;
    *out_ms = ms;
    return RAPID_OK;
}

}  // namespace rapid

using namespace rapid;

extern "C" {

int32_t rapid_view_overlay_spectrum(const rapid_view* v, uint64_t seed, double tol, int32_t max_steps, double* lambda2, double* lambda_min,
                                    double* residual, int32_t* steps, float* device_ms) {
    if (!v) { set_error("NULL view"); return RAPID_EINVAL; }
    if (!(tol > 0.0)) { set_error("tol must be positive"); return RAPID_EINVAL; }
    if (max_steps < 2 || max_steps > RAPID_OVERLAY_MAX_STEPS) { set_error("max_steps must be in [2, %d], got %d", RAPID_OVERLAY_MAX_STEPS, max_steps); return RAPID_EINVAL; }
    if (v->n < 3) { set_error("the overlay of %lld member(s) has no spectrum below 2K to report (3 or more are needed)", (long long)v->n); return RAPID_EINVAL; }
    DeviceGuard g(v->device);
    Ritz r = {0.0, 0.0, 0.0};
    int32_t m = 0;
    float ms = 0.f;
    RAPID_CHECK(overlay_spectrum(v, seed, tol, max_steps, &r, &m, &ms));
    if (lambda2) *lambda2 = r.hi;
    if (lambda_min) *lambda_min = r.lo;
    if (residual) *residual = r.residual;
    if (steps) *steps = m;
    if (device_ms) *device_ms = ms;
    return RAPID_OK;
}

}  // extern "C"
