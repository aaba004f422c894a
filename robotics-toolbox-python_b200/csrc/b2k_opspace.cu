// b2k_opspace.cu -- operational-space dynamics: the arithmetic of the reference's DynamicsMixin.inertia_x, coriolis_x,
// gravload_x and accel_x (robot/Dynamics.py, between gravload and itorque), which loop over rows in Python with
// numpy inv / pinv and triple products.  The joint-space quantities (M, C, G, the analytical Jacobian and its time
// derivative) come from the existing kernels; this file is the epilogue over their outputs.
//
// One lane per row, blocks of one warp.  Every array moves through a per-warp shared-memory tile (32 rows) so that the
// global loads and stores are coalesced, as in the lane-per-row kernels of b2k_extra.cu.  Ji (n x 6) is formed once per
// row and kept in registers; M, C and Jd are then streamed one row at a time from the tile against it, so the largest
// live set is Ji + one 6x6 accumulator (42 + 36 doubles at n = 7).  Mx, which Cx needs after C has replaced M in the
// tile, waits in a per-lane slot of shared memory instead of registers.
#include <math_constants.h>

#include "b2k_common.cuh"

struct OpsArgs {
    const void *Ja, *Ji_in, *M, *C, *Jd, *G, *Mx_in, *xd, *w;
    void *Ji, *Mx, *Cx, *Gx, *qd, *tau;
    long long nrows;
};

template <typename real>
__device__ __forceinline__ void ops_stage_in(real *t, const void *g, long long row0, int rows, int E, int lane)
{
    __syncwarp(); // every lane is done with what the tile held
    const real *src = (const real *)g + row0 * E;
    for (int e = lane; e < rows * E; e += 32) t[e] = src[e];
    __syncwarp();
}

template <typename real, int E>
__device__ __forceinline__ void ops_stage_out(real *t, void *g, long long row0, int rows, int lane, const real (&v)[E])
{
    __syncwarp();
    if (lane < rows) {
#pragma unroll
        for (int k = 0; k < E; k++) t[lane * E + k] = v[k];
    }
    __syncwarp();
    real *dst = (real *)g + row0 * E;
    for (int e = lane; e < rows * E; e += 32) dst[e] = t[e];
}

// x = inv(a) for a 6x6 row-major matrix: Gauss-Jordan with partial pivoting.  The pivot of column c is the first row
// of largest magnitude at or below c -- the choice LAPACK getrf (numpy.linalg.inv) makes, since eliminating above the
// pivot does not change the rows below it.  The row swap is a chain of predicated exchanges with compile-time indices,
// so both matrices stay in registers.  Returns false on an exactly zero pivot (numpy raises LinAlgError there).
template <typename real>
__device__ __forceinline__ bool ops_inv6(const real (&a)[36], real (&x)[36])
{
    real A[36];
    bool ok = true;
#pragma unroll
    for (int e = 0; e < 36; e++) { A[e] = a[e]; x[e] = (e / 6 == e % 6) ? (real)1 : (real)0; }
#pragma unroll
    for (int c = 0; c < 6; c++) {
        int p = c;
        real best = fabs(A[c * 6 + c]);
#pragma unroll
        for (int r = c + 1; r < 6; r++) {
            const real v = fabs(A[r * 6 + c]);
            if (v > best) { best = v; p = r; }
        }
        ok = ok && best != (real)0;
#pragma unroll
        for (int r = c + 1; r < 6; r++) {
            if (r == p) {
#pragma unroll
                for (int k = c; k < 6; k++) { const real t = A[c * 6 + k]; A[c * 6 + k] = A[r * 6 + k]; A[r * 6 + k] = t; }
#pragma unroll
                for (int k = 0; k < 6; k++) { const real t = x[c * 6 + k]; x[c * 6 + k] = x[r * 6 + k]; x[r * 6 + k] = t; }
            }
        }
        const real ip = (real)1 / A[c * 6 + c];
#pragma unroll
        for (int k = c + 1; k < 6; k++) A[c * 6 + k] *= ip;
#pragma unroll
        for (int k = 0; k < 6; k++) x[c * 6 + k] *= ip;
#pragma unroll
        for (int r = 0; r < 6; r++) {
            if (r == c) continue;
            const real f = A[r * 6 + c];
#pragma unroll
            for (int k = c + 1; k < 6; k++) A[r * 6 + k] = fma(-f, A[c * 6 + k], A[r * 6 + k]);
#pragma unroll
            for (int k = 0; k < 6; k++) x[r * 6 + k] = fma(-f, x[c * 6 + k], x[r * 6 + k]);
        }
    }
    return ok;
}

// ji = pinv(a), a = Ja (6 x N row-major), ji (N x 6 row-major).  One-sided Jacobi SVD -- the iteration of k_singular_all
// in b2k_extra.cu -- on the thinner orientation W (P x D, D = min(6, N) columns) with the rotations accumulated in V:
// W_final = W0 V, column k of W_final = s_k times a left singular vector.  Then pinv = sum_k (1 / s_k^2) x_k y_k^T over
// the singular values numpy keeps (s_k > 1e-15 s_max, numpy.linalg.pinv's default rcond); x_k / y_k are the columns of
// V / W_final (tall Ja) or W_final / V (wide Ja).
template <typename real, int N>
__device__ __forceinline__ void ops_pinv(const real (&a)[6 * N], real (&ji)[N * 6])
{
    constexpr bool tall = N <= 6;
    constexpr int P = tall ? 6 : N, D = tall ? N : 6;
    real W[P * D], V[D * D];
#pragma unroll
    for (int r = 0; r < P; r++)
#pragma unroll
        for (int c = 0; c < D; c++) W[r * D + c] = tall ? a[r * N + c] : a[c * N + r];
#pragma unroll
    for (int e = 0; e < D * D; e++) V[e] = (e / D == e % D) ? (real)1 : (real)0;
    const real eps = sizeof(real) == 8 ? (real)1e-15 : (real)1e-6;
#pragma unroll 1
    for (int sweep = 0; sweep < 30; sweep++) {
        bool rotated = false;
#pragma unroll
        for (int p = 0; p < D - 1; p++)
#pragma unroll
            for (int q = p + 1; q < D; q++) {
                real al = 0, be = 0, ga = 0;
#pragma unroll
                for (int r = 0; r < P; r++) {
                    const real x = W[r * D + p], y = W[r * D + q];
                    al = fma(x, x, al); be = fma(y, y, be); ga = fma(x, y, ga);
                }
                const bool skip = fabs(ga) <= eps * sqrt(al * be) || ga == 0;
                rotated = rotated || !skip;
                const real zeta = (be - al) / (2 * (skip ? (real)1 : ga));
                const real t = (zeta >= 0 ? (real)1 : (real)-1) / (fabs(zeta) + sqrt(1 + zeta * zeta));
                const real c0 = 1 / sqrt(1 + t * t);
                const real cs = skip ? (real)1 : c0, sn = skip ? (real)0 : c0 * t;
#pragma unroll
                for (int r = 0; r < P; r++) {
                    const real x = W[r * D + p], y = W[r * D + q];
                    W[r * D + p] = cs * x - sn * y;
                    W[r * D + q] = sn * x + cs * y;
                }
#pragma unroll
                for (int r = 0; r < D; r++) {
                    const real x = V[r * D + p], y = V[r * D + q];
                    V[r * D + p] = cs * x - sn * y;
                    V[r * D + q] = sn * x + cs * y;
                }
            }
        if (!rotated) break;
    }
    real inv2[D], s2max = 0;
#pragma unroll
    for (int c = 0; c < D; c++) {
        real nn = 0;
#pragma unroll
        for (int r = 0; r < P; r++) nn = fma(W[r * D + c], W[r * D + c], nn);
        inv2[c] = nn;
        s2max = fmax(s2max, nn);
    }
    const real cut = (real)1e-15 * sqrt(s2max);
#pragma unroll
    for (int c = 0; c < D; c++) inv2[c] = sqrt(inv2[c]) > cut ? (real)1 / inv2[c] : (real)0;
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < 6; j++) {
            real s = 0;
#pragma unroll
            for (int k = 0; k < D; k++) s = tall ? fma(V[i * D + k] * inv2[k], W[j * D + k], s) : fma(W[i * D + k] * inv2[k], V[j * D + k], s);
            ji[i * 6 + j] = s;
        }
}

// acc (6x6) = Ji^T X Ji with X (N x N) the lane's row of the tile, streamed one row of X at a time
template <typename real, int N>
__device__ __forceinline__ void ops_congruence(const real *X, const real (&ji)[N * 6], real (&acc)[36])
{
#pragma unroll
    for (int e = 0; e < 36; e++) acc[e] = 0;
#pragma unroll
    for (int i = 0; i < N; i++) {
        real t[6] = {0, 0, 0, 0, 0, 0}; // row i of X Ji
#pragma unroll
        for (int j = 0; j < N; j++) {
            const real x = X[i * N + j];
#pragma unroll
            for (int b = 0; b < 6; b++) t[b] = fma(x, ji[j * 6 + b], t[b]);
        }
#pragma unroll
        for (int a = 0; a < 6; a++)
#pragma unroll
            for (int b = 0; b < 6; b++) acc[a * 6 + b] = fma(ji[i * 6 + a], t[b], acc[a * 6 + b]);
    }
}

template <typename real, int N, bool INV>
__global__ void __launch_bounds__(32) k_opspace(const __grid_constant__ OpsArgs A)
{
    constexpr int S = (6 * N > N * N ? 6 * N : N * N) > 36 ? (6 * N > N * N ? 6 * N : N * N) : 36;
    constexpr int MXS = 37; // odd pitch of the per-lane Mx slot
    __shared__ real tile[32 * S];
    __shared__ real mxs[32 * MXS];
    const int lane = threadIdx.x;
    const long long row0 = (long long)blockIdx.x * 32;
    const int rows = (int)(A.nrows - row0 < 32 ? A.nrows - row0 : 32);
    const int lr = lane < rows ? lane : 0; // idle lanes of a ragged tile recompute row 0 and store nothing

    real ji[N * 6];
    if (A.Ja && (!A.Ji_in || A.tau)) {
        real a[6 * N];
        ops_stage_in<real>(tile, A.Ja, row0, rows, 6 * N, lane);
#pragma unroll
        for (int e = 0; e < 6 * N; e++) a[e] = tile[lr * 6 * N + e];
        if (A.tau) { // tau = Ja^T w
            real tau[N];
            ops_stage_in<real>(tile, A.w, row0, rows, 6, lane);
#pragma unroll
            for (int i = 0; i < N; i++) {
                real s = 0;
#pragma unroll
                for (int r = 0; r < 6; r++) s = fma(a[r * N + i], tile[lr * 6 + r], s);
                tau[i] = s;
            }
            ops_stage_out<real, N>(tile, A.tau, row0, rows, lane, tau);
        }
        if (!A.Ji_in) {
            if constexpr (INV) {
                static_assert(N == 6, "the inverse needs a square Jacobian");
                if (!ops_inv6<real>(a, ji)) {
#pragma unroll
                    for (int e = 0; e < 36; e++) ji[e] = (real)CUDART_NAN;
                }
            } else {
                ops_pinv<real, N>(a, ji);
            }
        }
    }
    if (A.Ji_in) {
        ops_stage_in<real>(tile, A.Ji_in, row0, rows, 6 * N, lane);
#pragma unroll
        for (int e = 0; e < 6 * N; e++) ji[e] = tile[lr * 6 * N + e];
    }
    if (A.Ji) ops_stage_out<real, 6 * N>(tile, A.Ji, row0, rows, lane, ji);

    if (A.qd) { // qd = Ji xd
        real v[N];
        ops_stage_in<real>(tile, A.xd, row0, rows, 6, lane);
#pragma unroll
        for (int i = 0; i < N; i++) {
            real s = 0;
#pragma unroll
            for (int j = 0; j < 6; j++) s = fma(ji[i * 6 + j], tile[lr * 6 + j], s);
            v[i] = s;
        }
        ops_stage_out<real, N>(tile, A.qd, row0, rows, lane, v);
    }

    real *mx_slot = mxs + lane * MXS;
    if (A.Mx || (A.Cx && !A.Mx_in)) { // Mx = Ji^T M Ji
        real mx[36];
        ops_stage_in<real>(tile, A.M, row0, rows, N * N, lane);
        ops_congruence<real, N>(tile + lr * N * N, ji, mx);
        if (A.Cx) {
#pragma unroll
            for (int e = 0; e < 36; e++) mx_slot[e] = mx[e];
        }
        if (A.Mx) ops_stage_out<real, 36>(tile, A.Mx, row0, rows, lane, mx);
    } else if (A.Cx) {
        ops_stage_in<real>(tile, A.Mx_in, row0, rows, 36, lane);
#pragma unroll
        for (int e = 0; e < 36; e++) mx_slot[e] = tile[lr * 36 + e];
    }

    if (A.Cx) { // Cx = Ji^T C Ji - Mx (Jd Ji)
        real cx[36];
        ops_stage_in<real>(tile, A.C, row0, rows, N * N, lane);
        ops_congruence<real, N>(tile + lr * N * N, ji, cx);
        ops_stage_in<real>(tile, A.Jd, row0, rows, 6 * N, lane);
        const real *jd = tile + lr * 6 * N;
#pragma unroll
        for (int c = 0; c < 6; c++) {
            real e[6] = {0, 0, 0, 0, 0, 0}; // row c of Jd Ji
#pragma unroll
            for (int k = 0; k < N; k++) {
                const real d = jd[c * N + k];
#pragma unroll
                for (int b = 0; b < 6; b++) e[b] = fma(d, ji[k * 6 + b], e[b]);
            }
#pragma unroll
            for (int a = 0; a < 6; a++) {
                const real m = mx_slot[a * 6 + c];
#pragma unroll
                for (int b = 0; b < 6; b++) cx[a * 6 + b] = fma(-m, e[b], cx[a * 6 + b]);
            }
        }
        ops_stage_out<real, 36>(tile, A.Cx, row0, rows, lane, cx);
    }

    if (A.Gx) { // Gx = Ji^T G
        real gx[6];
        ops_stage_in<real>(tile, A.G, row0, rows, N, lane);
#pragma unroll
        for (int a = 0; a < 6; a++) {
            real s = 0;
#pragma unroll
            for (int i = 0; i < N; i++) s = fma(ji[i * 6 + a], tile[lr * N + i], s);
            gx[a] = s;
        }
        ops_stage_out<real, 6>(tile, A.Gx, row0, rows, lane, gx);
    }
}

// xdd = Ja qdd + Jd qd, the last stage of accel_x
template <typename real, int N>
__global__ void __launch_bounds__(32) k_opspace_xdd(const real *__restrict__ Ja, const real *__restrict__ qdd,
                                                    const real *__restrict__ Jd, const real *__restrict__ qd, long long nrows,
                                                    real *__restrict__ xdd)
{
    __shared__ real tile[32 * 6 * N];
    __shared__ real vec[32 * N];
    const int lane = threadIdx.x;
    const long long row0 = (long long)blockIdx.x * 32;
    const int rows = (int)(nrows - row0 < 32 ? nrows - row0 : 32);
    const int lr = lane < rows ? lane : 0;
    real x[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int pass = 0; pass < 2; pass++) {
        ops_stage_in<real>(tile, pass == 0 ? (const void *)Ja : (const void *)Jd, row0, rows, 6 * N, lane);
        ops_stage_in<real>(vec, pass == 0 ? (const void *)qdd : (const void *)qd, row0, rows, N, lane);
#pragma unroll
        for (int r = 0; r < 6; r++)
#pragma unroll
            for (int k = 0; k < N; k++) x[r] = fma(tile[lr * 6 * N + r * N + k], vec[lr * N + k], x[r]);
    }
    ops_stage_out<real, 6>(tile, xdd, row0, rows, lane, x);
}

template <typename real>
static int opspace_launch(int n, int inverse, const OpsArgs &A, cudaStream_t st)
{
    const unsigned blocks = (unsigned)((A.nrows + 31) / 32);
    if (inverse == 0) {
        k_opspace<real, 6, true><<<blocks, 32, 0, st>>>(A);
    } else {
        switch (n) {
#define B2K_CASE(NN) \
    case NN: k_opspace<real, NN, false><<<blocks, 32, 0, st>>>(A); break;
            B2K_CASE(1) B2K_CASE(2) B2K_CASE(3) B2K_CASE(4) B2K_CASE(5)
            B2K_CASE(6) B2K_CASE(7) B2K_CASE(8) B2K_CASE(9) B2K_CASE(10)
#undef B2K_CASE
        }
    }
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

template <typename real>
static int opspace_xdd_launch(int n, const void *Ja, const void *qdd, const void *Jd, const void *qd, long long N, void *xdd,
                              cudaStream_t st)
{
    const unsigned blocks = (unsigned)((N + 31) / 32);
    switch (n) {
#define B2K_CASE(NN)                                                                                                   \
    case NN:                                                                                                           \
        k_opspace_xdd<real, NN><<<blocks, 32, 0, st>>>((const real *)Ja, (const real *)qdd, (const real *)Jd,        \
                                                        (const real *)qd, N, (real *)xdd);                            \
        break;
        B2K_CASE(1) B2K_CASE(2) B2K_CASE(3) B2K_CASE(4) B2K_CASE(5)
        B2K_CASE(6) B2K_CASE(7) B2K_CASE(8) B2K_CASE(9) B2K_CASE(10)
#undef B2K_CASE
    }
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

extern "C" int b2k_opspace(int dtype, int n, int inverse, const void *Ja, const void *Ji_in, const void *M, const void *Cm,
                           const void *Jd, const void *G, const void *Mx_in, const void *xd, const void *w, int64_t N, void *Ji,
                           void *Mx, void *Cx, void *Gx, void *qd, void *tau, void *stream)
{
    const char *fn = "b2k_opspace";
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (n < 1 || n > B2K_MAX_JOINTS) { b2k_set_error("%s: n must be 1..%d", fn, B2K_MAX_JOINTS); return B2K_ERR_INVALID; }
    if (inverse != B2K_OPS_INV && inverse != B2K_OPS_PINV) {
        b2k_set_error("%s: inverse must be B2K_OPS_INV (0) or B2K_OPS_PINV (1)", fn);
        return B2K_ERR_INVALID;
    }
    if (inverse == B2K_OPS_INV && n != 6) {
        b2k_set_error("%s: inv needs a square analytical Jacobian (n = 6), got n = %d; use the pseudo-inverse", fn, n);
        return B2K_ERR_INVALID;
    }
    if (N < 0) { b2k_set_error("%s: bad N", fn); return B2K_ERR_INVALID; }
    if (!Ji && !Mx && !Cx && !Gx && !qd && !tau) { b2k_set_error("%s: no output requested", fn); return B2K_ERR_INVALID; }
    if ((Ji || Mx || Cx || Gx || qd) && !Ja && !Ji_in) { b2k_set_error("%s: Ji, Mx, Cx, Gx and qd need Ja or a given Ji (both NULL)", fn); return B2K_ERR_INVALID; }
    if (Mx && !M) { b2k_set_error("%s: Mx needs M (NULL)", fn); return B2K_ERR_INVALID; }
    if (Cx && (!Cm || !Jd || (!M && !Mx_in))) { b2k_set_error("%s: Cx needs C, Jd and M or a given Mx (NULL)", fn); return B2K_ERR_INVALID; }
    if (Gx && !G) { b2k_set_error("%s: Gx needs G (NULL)", fn); return B2K_ERR_INVALID; }
    if (qd && !xd) { b2k_set_error("%s: qd needs xd (NULL)", fn); return B2K_ERR_INVALID; }
    if (tau && (!Ja || !w)) { b2k_set_error("%s: tau needs Ja and w (NULL)", fn); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(Ja ? Ja : Ji_in);
    OpsArgs A;
    A.Ja = Ja; A.Ji_in = Ji_in; A.M = M; A.C = Cm; A.Jd = Jd; A.G = G; A.Mx_in = Mx_in; A.xd = xd; A.w = w;
    A.Ji = Ji; A.Mx = Mx; A.Cx = Cx; A.Gx = Gx; A.qd = qd; A.tau = tau;
    A.nrows = N;
    return dtype == B2K_F64 ? opspace_launch<double>(n, inverse, A, (cudaStream_t)stream)
                            : opspace_launch<float>(n, inverse, A, (cudaStream_t)stream);
}

extern "C" int b2k_opspace_xdd(int dtype, int n, const void *Ja, const void *qdd, const void *Jd, const void *qd, int64_t N,
                               void *xdd, void *stream)
{
    const char *fn = "b2k_opspace_xdd";
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (n < 1 || n > B2K_MAX_JOINTS) { b2k_set_error("%s: n must be 1..%d", fn, B2K_MAX_JOINTS); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: bad N", fn); return B2K_ERR_INVALID; }
    if (N > 0 && (!Ja || !qdd || !Jd || !qd || !xdd)) { b2k_set_error("%s: Ja, qdd, Jd, qd and xdd must not be NULL", fn); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(Ja);
    return dtype == B2K_F64 ? opspace_xdd_launch<double>(n, Ja, qdd, Jd, qd, N, xdd, (cudaStream_t)stream)
                            : opspace_xdd_launch<float>(n, Ja, qdd, Jd, qd, N, xdd, (cudaStream_t)stream);
}
