// b2k_extra.cu -- pure functions of the Jacobian (SURVEY 8f-2): manipulator Hessian, Yoshikawa
// manipulability, Jacobian time derivative and manipulability Jacobian.  Replaces fknm.ETS_hessian0 /
// ETS_hessiane (reference fknm.cpp:583-783 -> _ETS_hessian methods.cpp:16-32), the yoshikawa branch of
// ETS.manipulability (ETS.py:1780-1787), Robot.jacob0_dot (Robot.py:964-1099) and ETS.jacobm (ETS.py:1628-1685).
#include "b2k_common.cuh"
#include "b2k_ik.cuh" // ik_angle_axis

// H[a, 0:3, b] = Jw_a x Jv_b, H[a, 3:6, b] = Jw_a x Jw_b for b >= a; mirrored translational block and a zero
// rotational block for b < a (methods.cpp:18-31).  A store stream: 6 n^2 outputs per row against 6 n inputs.
// One warp per row; the 6n values of J sit in shared memory (slot 6n holds a zero) and lane l produces the output pairs
// l, l + 32, ... of the row.  Which four J entries an output needs depends only on its position in the row, i.e. on
// (lane, iteration): the shared-memory offsets are worked out ONCE per thread and kept in registers, so a row costs
// 8 LDS + 4 flops + one vector store per pair and no index arithmetic (the previous form decoded (a, r, b) and
// branched per element: ~40 instructions per output, issue-bound; one thread per output
// element with J through L1 was slower still).  The next row's J values are fetched while this one is written.
template <typename real> struct Pair2;
template <> struct Pair2<double> { typedef double2 type; };
template <> struct Pair2<float> { typedef float2 type; };

template <typename real, int N>
__global__ void __launch_bounds__(256) k_hessian(const real *__restrict__ J, long long nrows, real *__restrict__ H, int vec_ok)
{
    constexpr int E = 6 * N, PAIRS = 3 * N * N, IT = (PAIRS + 31) / 32, LD = (E + 31) / 32;
    typedef typename Pair2<real>::type real2;
    __shared__ real sJ[8][E + 2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    real *j = sJ[warp];
    if (lane == 0) j[E] = 0;

    // per-thread table: shared-memory slots of (u1, u2, w1, w2) for both elements of each of this lane's pairs
    unsigned short ix[IT][2][4];
#pragma unroll
    for (int i = 0; i < IT; i++)
#pragma unroll
        for (int k = 0; k < 2; k++) {
            const int e = 2 * (lane + 32 * i) + k;
            const int a = e / E, r = (e / N) % 6, b = e % N;
            const bool live = e < 6 * N * N && (b >= a || r < 3);
            // u x w, component c: u = Jw of the lower-numbered joint, w = Jv (r < 3) or Jw (r >= 3) of the other
            const int lo = b >= a ? a : b, hi = b >= a ? b : a;
            const int c = r % 3, c1 = (c + 1) % 3, c2 = (c + 2) % 3, wrow = r < 3 ? 0 : 3;
            ix[i][k][0] = live ? (3 + c1) * N + lo : E;
            ix[i][k][1] = live ? (3 + c2) * N + lo : E;
            ix[i][k][2] = live ? (wrow + c1) * N + hi : E;
            ix[i][k][3] = live ? (wrow + c2) * N + hi : E;
        }

    const long long wstride = (long long)gridDim.x * 8;
    long long row = (long long)blockIdx.x * 8 + warp;
    real nx[LD];
#pragma unroll
    for (int t = 0; t < LD; t++) nx[t] = (row < nrows && lane + 32 * t < E) ? J[row * E + lane + 32 * t] : (real)0;
    for (; row < nrows; row += wstride) {
#pragma unroll
        for (int t = 0; t < LD; t++)
            if (lane + 32 * t < E) j[lane + 32 * t] = nx[t];
        __syncwarp();
        const long long nrow = row + wstride;
#pragma unroll
        for (int t = 0; t < LD; t++)
            if (nrow < nrows && lane + 32 * t < E) nx[t] = J[nrow * E + lane + 32 * t];
        real *out = H + row * (6 * N * N);
#pragma unroll
        for (int i = 0; i < IT; i++) {
            const int p = lane + 32 * i;
            const real v0 = j[ix[i][0][0]] * j[ix[i][0][3]] - j[ix[i][0][1]] * j[ix[i][0][2]];
            const real v1 = j[ix[i][1][0]] * j[ix[i][1][3]] - j[ix[i][1][1]] * j[ix[i][1][2]];
            if (i < IT - 1 || p < PAIRS) {
                if (vec_ok) {
                    real2 v; v.x = v0; v.y = v1;
                    reinterpret_cast<real2 *>(out)[p] = v;
                } else {
                    out[2 * p] = v0; out[2 * p + 1] = v1;
                }
            }
        }
        __syncwarp();
    }
}

// The same Hessian for output arrays that are 16-byte aligned (every torch allocation): a LANE per row, the row's J in
// registers, every output a compile-time choice of four registers -- no shared-memory operand reads at all (the kernel
// above spends 8 LDS.64 per output pair, 3.2 bank cycles each: shared-memory bandwidth, not HBM, bounds it).
// A block of 4 warps owns a tile of 32 rows; warp w produces the 16-byte units w, w + 4, ... of every row and stores
// them into a shared-memory image of the tile's output block, which leaves through the TMA engine
// (cp.async.bulk shared -> global: no LDS / STG instructions).  The row pitch of the image is an odd number of units,
// so the lane-per-row vector stores are bank-conflict free: where the row itself is an odd number of units the image is
// exact and ONE bulk copy moves the tile; otherwise a 16-byte pad follows each row and the lane that owns a row issues
// its copy.  One-shot grid (a tile per block), 3 resident blocks per SM at n = 7 fp64 (75 KB of image each): while one
// block's image drains the others compute.
template <typename real, int N> struct HessTile {
    static constexpr int E = 6 * N;
    static constexpr int U = (sizeof(real) == 8 || N % 2 == 0) ? 16 : 8; // bytes per unit
    static constexpr int EPU = U / (int)sizeof(real);                    // elements per unit
    static constexpr int ROWB = 6 * N * N * (int)sizeof(real);
    static constexpr int RU = ROWB / U;  // units per row
    static constexpr int PU = RU | 1;    // pitch in units (odd)
    static constexpr bool EXACT = PU == RU;
    static constexpr int SMEM = 32 * PU * U;
    static_assert(ROWB % U == 0, "row is a whole number of units");
    static_assert(32 * E * (int)sizeof(real) <= SMEM, "the J tile fits in front of the image");
};

template <typename real, int N>
__device__ __forceinline__ real hess_elem(const real (&j)[6 * N], int e)
{
    const int a = e / (6 * N), r = (e / N) % 6, b = e % N;
    if (!(b >= a || r < 3)) return (real)0;
    const int lo = b >= a ? a : b, hi = b >= a ? b : a;
    const int c = r % 3, c1 = (c + 1) % 3, c2 = (c + 2) % 3, wrow = r < 3 ? 0 : 3;
    return j[(3 + c1) * N + lo] * j[(wrow + c2) * N + hi] - j[(3 + c2) * N + lo] * j[(wrow + c1) * N + hi];
}

template <typename real, int N, int W>
__device__ __forceinline__ void hess_units(const real (&j)[6 * N], unsigned char *rowimg)
{
    typedef HessTile<real, N> HT;
#pragma unroll
    for (int u = W; u < HT::RU; u += 4) {
        real v[HT::EPU];
#pragma unroll
        for (int k = 0; k < HT::EPU; k++) v[k] = hess_elem<real, N>(j, u * HT::EPU + k);
        if constexpr (HT::U == 16 && sizeof(real) == 8) {
            *reinterpret_cast<double2 *>(rowimg + u * 16) = make_double2(v[0], v[1]);
        } else if constexpr (HT::U == 16) {
            *reinterpret_cast<float4 *>(rowimg + u * 16) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
            *reinterpret_cast<float2 *>(rowimg + u * 8) = make_float2(v[0], v[1]);
        }
    }
}

template <typename real, int N>
__global__ void __launch_bounds__(128) k_hessian_tile(const real *__restrict__ J, long long nrows, real *__restrict__ H)
{
    typedef HessTile<real, N> HT;
    extern __shared__ __align__(16) unsigned char hess_img[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long row0 = (long long)blockIdx.x * 32;
    const int rows = (int)(nrows - row0 < 32 ? nrows - row0 : 32);

    // the tile's J block (contiguous) -> front of the image, coalesced; then a lane takes its row into registers
    {
        real *sj = reinterpret_cast<real *>(hess_img);
        const real *g = J + row0 * HT::E;
        for (int e = threadIdx.x; e < rows * HT::E; e += 128) sj[e] = g[e];
    }
    __syncthreads();
    real j[HT::E];
    {
        const real *sj = reinterpret_cast<const real *>(hess_img) + lane * HT::E;
#pragma unroll
        for (int e = 0; e < HT::E; e++) j[e] = sj[e];
    }
    __syncthreads(); // the image overwrites the J tile

    unsigned char *rowimg = hess_img + (size_t)lane * (HT::PU * HT::U);
    switch (warp) {
    case 0: hess_units<real, N, 0>(j, rowimg); break;
    case 1: hess_units<real, N, 1>(j, rowimg); break;
    case 2: hess_units<real, N, 2>(j, rowimg); break;
    default: hess_units<real, N, 3>(j, rowimg); break;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    real *gout = H + row0 * (6 * N * N);
    if constexpr (HT::EXACT) {
        const unsigned bytes = (unsigned)rows * HT::ROWB;
        if ((bytes & 15u) == 0) {
            if (threadIdx.x == 0) {
                const unsigned sa = (unsigned)__cvta_generic_to_shared(hess_img);
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gout), "r"(sa), "r"(bytes) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            }
        } else { // ragged last tile of an fp32 / odd-n array whose byte count is 8 mod 16
            const real *img = reinterpret_cast<const real *>(hess_img);
            for (int e = threadIdx.x; e < rows * 6 * N * N; e += 128) gout[e] = img[e];
        }
    } else {
        if (threadIdx.x < rows) {
            const unsigned sa = (unsigned)__cvta_generic_to_shared(rowimg);
            const unsigned bytes = HT::ROWB;
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gout + (size_t)lane * (6 * N * N)), "r"(sa), "r"(bytes) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        }
    }
}

// ---- lane-per-row kernels over Jacobian rows: 64-thread blocks, each warp stages its tile of 32 rows (6N reals each)
// through shared memory so that the global loads / stores are coalesced, and a lane then owns one row in registers.
// (Reading the rows straight from global memory -- 32 lanes x a 6N-real stride per load instruction -- measured
// a small fraction of the HBM rate.)
#define B2K_XT 64 /* threads per block of the staged kernels: 2 warps x 32 x 60 doubles = 30 KB at n = 10 */
template <typename real>
__device__ __forceinline__ void xt_copy(real *dst, const real *src, int count, int lane)
{
    for (int e = lane; e < count; e += 32) dst[e] = src[e];
}

// Yoshikawa measure with all six axes selected and n > 6 (the Gram matrix J J^T is 6 x 6 SPD): m = prod L_jj.
template <typename real, int N>
__global__ void __launch_bounds__(B2K_XT) k_yoshikawa_all(const real *__restrict__ J, long long nrows, real *__restrict__ m)
{
    __shared__ real tile[B2K_XT / 32][32 * 6 * N];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long row0 = ((long long)blockIdx.x * (B2K_XT / 32) + warp) * 32;
    if (row0 >= nrows) return;
    const int rows = (int)(nrows - row0 < 32 ? nrows - row0 : 32);
    xt_copy(tile[warp], J + row0 * (6 * N), rows * 6 * N, lane);
    __syncwarp();
    if (lane >= rows) return;
    const real *j = tile[warp] + lane * (6 * N);
    real A[21];
#pragma unroll
    for (int a = 0; a < 6; a++)
#pragma unroll
        for (int b = 0; b <= a; b++) {
            real s = 0;
#pragma unroll
            for (int k = 0; k < N; k++) s = fma(j[a * N + k], j[b * N + k], s);
            A[a * (a + 1) / 2 + b] = s;
        }
    const bool ok = ik_chol_factor<real, 6>(A);
    real p = 1;
#pragma unroll
    for (int a = 0; a < 6; a++) p *= A[a * (a + 1) / 2 + a]; // 1 / L_aa
    m[row0 + lane] = ok ? (real)1 / p : (real)0; // a rank-deficient J: det(J J^T) = 0 up to rounding
}

// Jd = sum_i H[i] qd[i]  (Robot.jacob0_dot, Robot.py:964-1099: np.tensordot(H, qd, (0, 0))) without materialising H:
// Jd[r, b] = sum_a qd[a] * H[a, r, b], H from J as in k_hessian (methods.cpp:16-32).  One lane per row, J and qd in
// registers, the tile doubling as the output stage.  (The first version, a warp per row over shared memory, was slower.)
template <typename real, int N>
__global__ void __launch_bounds__(B2K_XT) k_jacob_dot_lane(const real *__restrict__ J, const real *__restrict__ qd, long long nrows,
                                                           real *__restrict__ Jd)
{
    __shared__ real tile[B2K_XT / 32][32 * 6 * N];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long row0 = ((long long)blockIdx.x * (B2K_XT / 32) + warp) * 32;
    if (row0 >= nrows) return;
    const int rows = (int)(nrows - row0 < 32 ? nrows - row0 : 32);
    real *t = tile[warp];
    xt_copy(t, J + row0 * (6 * N), rows * 6 * N, lane);
    __syncwarp();
    real j[6 * N], v[N];
    const int lr = lane < rows ? lane : 0;
#pragma unroll
    for (int e = 0; e < 6 * N; e++) j[e] = t[lr * (6 * N) + e];
#pragma unroll
    for (int a = 0; a < N; a++) v[a] = qd[(row0 + lr) * N + a];
    __syncwarp(); // every lane has its row: the tile becomes the output stage
#pragma unroll
    for (int r = 0; r < 6; r++) {
        const int c = r % 3, c1 = (c + 1) % 3, c2 = (c + 2) % 3, wrow = r < 3 ? 0 : 3;
#pragma unroll
        for (int b = 0; b < N; b++) {
            real acc = 0;
#pragma unroll
            for (int a = 0; a < N; a++) {
                if (b >= a || r < 3) {
                    const int lo = b >= a ? a : b, hi = b >= a ? b : a;
                    acc = fma(v[a], fma(j[(3 + c1) * N + lo], j[(wrow + c2) * N + hi], -(j[(3 + c2) * N + lo] * j[(wrow + c1) * N + hi])), acc);
                }
            }
            if (lane < rows) t[lane * (6 * N) + r * N + b] = acc;
        }
    }
    __syncwarp();
    xt_copy(Jd + row0 * (6 * N), t, rows * 6 * N, lane);
}

// m = sqrt(|det(Ja Ja^T)|) with Ja = the selected rows of J (|det Ja| when Ja is square), ETS.py:1780-1787
template <typename real, int N>
__global__ void __launch_bounds__(128) k_yoshikawa(const real *__restrict__ J, long long nrows, unsigned axes_mask,
                                                   real *__restrict__ m)
{
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    int sel[6], na = 0;
    for (int k = 0; k < 6; k++)
        if (axes_mask & (1u << k)) sel[na++] = k;
    real A[36];
    const real *j = J + row * (6 * N);
    const bool square = (na == N);
    for (int a = 0; a < na; a++)
        for (int b = 0; b < na; b++) {
            real s = 0;
            if (square) s = j[sel[a] * N + b];
            else
                for (int k = 0; k < N; k++) s += j[sel[a] * N + k] * j[sel[b] * N + k];
            A[a * na + b] = s;
        }
    real det = 1;
    for (int c = 0; c < na; c++) { // Gaussian elimination with partial pivoting
        int p = c;
        real best = fabs(A[c * na + c]);
        for (int r = c + 1; r < na; r++)
            if (fabs(A[r * na + c]) > best) { best = fabs(A[r * na + c]); p = r; }
        if (best == 0) { det = 0; break; }
        if (p != c) {
            for (int k = 0; k < na; k++) { real t = A[c * na + k]; A[c * na + k] = A[p * na + k]; A[p * na + k] = t; }
            det = -det;
        }
        det *= A[c * na + c];
        for (int r = c + 1; r < na; r++) {
            const real f = A[r * na + c] / A[c * na + c];
            for (int k = c + 1; k < na; k++) A[r * na + k] -= f * A[c * na + k];
        }
    }
    m[row] = square ? fabs(det) : sqrt(fabs(det));
}

// Manipulability Jacobian dm/dq (ETS.jacobm ETS.py:1628-1685, Robot.jacobm Robot.py:1124-1232):
//   Jm[i] = m * sum_{a,b} (Ja Ha_i^T)[a,b] * inv(Ja Ja^T)[a,b],  Ja / Ha = the selected Cartesian rows, m = Yoshikawa.
// One lane per row; the na x na Gram matrix is inverted by Gauss-Jordan with partial pivoting (its determinant
// gives m on the way).
// All six Cartesian axes selected (the default of ETS.jacobm): everything has compile-time indices and stays in
// registers.  The 6 x 6 Gram matrix A = J J^T is symmetric positive definite away from singularities: Cholesky (no
// pivot search, which would need run-time row indices -- i.e. local memory) gives m = sqrt(det A) = prod L_jj and the
// columns G[:, k] = A^-1 J[:, k]; then  sum_{a,b} (J H_i^T)[a,b] A^-1[a,b] = sum_{b,k} H_i[b,k] G[b,k]  (A^-1 is
// symmetric), which needs the Hessian terms once per (i, b, k) instead of once per (i, a, b, k): ~1 800 operations per
// row instead of ~14 000.  The Gram factor and the Hessian terms come from b2k_gram_chol6 / b2k_hess_term (b2k_ik.cuh),
// which the IK null-space term shares.  The general kernel below (na read at run time, Gauss-Jordan with pivoting, every array in
// local memory) is far slower.
template <typename real, int N>
__global__ void __launch_bounds__(128) k_jacobm_all(const real *__restrict__ J, long long nrows, real *__restrict__ Jm)
{
    // (rows are read straight from global memory here: with ~250 live registers the staged form -- 64-thread blocks,
    // 10 KB of shared memory per warp -- measured slower)
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    const real *jr = J + row * (6 * N);
    real j[6 * N];
#pragma unroll
    for (int e = 0; e < 6 * N; e++) j[e] = jr[e];
    auto jx = [&](int a, int k) { return j[a * N + k]; };
    real A[21], m;
    b2k_gram_chol6<real, N>(jx, A, m); // a singular Gram matrix ends in inf / nan, as numpy's inv does in the reference
    real G[6 * N];
#pragma unroll
    for (int k = 0; k < N; k++) {
        real x[6];
#pragma unroll
        for (int a = 0; a < 6; a++) x[a] = j[a * N + k];
        ik_chol_subst<real, 6>(A, x);
#pragma unroll
        for (int a = 0; a < 6; a++) G[a * N + k] = x[a];
    }
#pragma unroll
    for (int i = 0; i < N; i++) {
        real acc = 0;
#pragma unroll
        for (int r = 0; r < 6; r++)
#pragma unroll
            for (int k = 0; k < N; k++)
                if (k >= i || r < 3) acc = fma(b2k_hess_term<real>(jx, i, r, k), G[r * N + k], acc);
        Jm[row * N + i] = m * acc;
    }
}

template <typename real, int N>
__global__ void __launch_bounds__(128) k_jacobm(const real *__restrict__ J, long long nrows, unsigned axes_mask,
                                                real *__restrict__ Jm)
{
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    int sel[6], na = 0;
    for (int k = 0; k < 6; k++)
        if (axes_mask & (1u << k)) sel[na++] = k;
    const real *jr = J + row * (6 * N);
    real j[6 * N];
    for (int e = 0; e < 6 * N; e++) j[e] = jr[e];
    real A[36], Bi[36];
    for (int a = 0; a < na; a++)
        for (int b = 0; b < na; b++) {
            real s = 0;
            for (int k = 0; k < N; k++) s += j[sel[a] * N + k] * j[sel[b] * N + k];
            A[a * na + b] = s;
            Bi[a * na + b] = (a == b) ? (real)1 : (real)0;
        }
    // m as k_yoshikawa computes it: |det Ja| for a square selection, sqrt|det(Ja Ja^T)| otherwise
    real det = 1;
    for (int c = 0; c < na; c++) {
        int p = c;
        real best = fabs(A[c * na + c]);
        for (int r = c + 1; r < na; r++)
            if (fabs(A[r * na + c]) > best) { best = fabs(A[r * na + c]); p = r; }
        if (p != c) {
            for (int k = 0; k < na; k++) {
                real t = A[c * na + k]; A[c * na + k] = A[p * na + k]; A[p * na + k] = t;
                t = Bi[c * na + k]; Bi[c * na + k] = Bi[p * na + k]; Bi[p * na + k] = t;
            }
            det = -det;
        }
        const real piv = A[c * na + c];
        det *= piv;
        const real inv = (real)1 / piv; // a singular Gram matrix gives inf/nan, as numpy's inv raises / returns garbage
        for (int k = 0; k < na; k++) { A[c * na + k] *= inv; Bi[c * na + k] *= inv; }
        for (int r = 0; r < na; r++) {
            if (r == c) continue;
            const real f = A[r * na + c];
            for (int k = 0; k < na; k++) { A[r * na + k] -= f * A[c * na + k]; Bi[r * na + k] -= f * Bi[c * na + k]; }
        }
    }
    const real m = sqrt(fabs(det));
    for (int i = 0; i < N; i++) {
        real acc = 0;
        for (int a = 0; a < na; a++)
            for (int b = 0; b < na; b++) {
                // c[a][b] = sum_k Ja[a][k] * H[i][sel b][k]
                const int r = sel[b], cc = r % 3, c1 = (cc + 1) % 3, c2 = (cc + 2) % 3, wrow = r < 3 ? 0 : 3;
                real cab = 0;
                for (int k = 0; k < N; k++) {
                    if (k >= i || r < 3) {
                        const int lo = k >= i ? i : k, hi = k >= i ? k : i;
                        const real u1 = j[(3 + c1) * N + lo], u2 = j[(3 + c2) * N + lo];
                        const real w1 = j[(wrow + c1) * N + hi], w2 = j[(wrow + c2) * N + hi];
                        cab += j[sel[a] * N + k] * (u1 * w2 - u2 * w1);
                    }
                }
                acc += cab * Bi[a * na + b];
            }
        Jm[row * N + i] = m * acc;
    }
}

// Singular-value measures of ETS.manipulability (ETS.py:1789-1796): "minsingular" = the smallest singular value of
// Ja = the selected rows of J (numpy svd(Ja)[-1]: min(rows, n) values), "invcondition" = 1 / cond(Ja) = s_min / s_max.
// One lane per row; one-sided (Hestenes) Jacobi on the thinner orientation of Ja (columns = min(rows, n) <= 6,
// length max(rows, n) <= 10): plane rotations make the columns mutually orthogonal, their norms are the singular
// values -- accurate to rounding even next to a singularity, where squaring into the Gram matrix would lose half the digits.
// All six axes selected: the shape of the working matrix (P x D = max(6,N) x min(6,N)) is known at compile time, every
// index is a constant, the 6N values live in registers (the general kernel below keeps them in local memory because its
// shape is read from the axes mask, far from what the traffic needs).
template <typename real, int N>
__global__ void __launch_bounds__(128) k_singular_all(const real *__restrict__ J, long long nrows, int kind, real *__restrict__ m)
{
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    constexpr bool tall = 6 >= N;
    constexpr int P = tall ? 6 : N, D = tall ? N : 6;
    const real *j = J + row * (6 * N);
    real W[P * D];
#pragma unroll
    for (int r = 0; r < P; r++)
#pragma unroll
        for (int c = 0; c < D; c++) W[r * D + c] = tall ? j[r * N + c] : j[c * N + r];
    const real eps = sizeof(real) == 8 ? (real)1e-15 : (real)1e-6;
#pragma unroll 1
    for (int sweep = 0; sweep < 30; sweep++) {
        bool rotated = false;
#pragma unroll
        for (int a = 0; a < D - 1; a++)
#pragma unroll
            for (int b = a + 1; b < D; b++) {
                real al = 0, be = 0, ga = 0;
#pragma unroll
                for (int r = 0; r < P; r++) {
                    const real x = W[r * D + a], y = W[r * D + b];
                    al = fma(x, x, al); be = fma(y, y, be); ga = fma(x, y, ga);
                }
                const bool skip = fabs(ga) <= eps * sqrt(al * be) || ga == 0;
                rotated = rotated || !skip;
                const real zeta = (be - al) / (2 * (skip ? (real)1 : ga));
                const real t = (zeta >= 0 ? (real)1 : (real)-1) / (fabs(zeta) + sqrt(1 + zeta * zeta));
                const real c0 = 1 / sqrt(1 + t * t);
                const real cs = skip ? (real)1 : c0, sn = skip ? (real)0 : c0 * t; // identity rotation where the pair is orthogonal
#pragma unroll
                for (int r = 0; r < P; r++) {
                    const real x = W[r * D + a], y = W[r * D + b];
                    W[r * D + a] = cs * x - sn * y;
                    W[r * D + b] = sn * x + cs * y;
                }
            }
        if (!rotated) break;
    }
    real smin = 0, smax = 0;
#pragma unroll
    for (int c = 0; c < D; c++) {
        real nn = 0;
#pragma unroll
        for (int r = 0; r < P; r++) nn = fma(W[r * D + c], W[r * D + c], nn);
        nn = sqrt(nn);
        if (c == 0 || nn < smin) smin = nn;
        if (c == 0 || nn > smax) smax = nn;
    }
    m[row] = kind == 0 ? smin : (smax > 0 ? smin / smax : (real)0);
}

template <typename real, int N>
__global__ void __launch_bounds__(128) k_singular(const real *__restrict__ J, long long nrows, unsigned axes_mask, int kind,
                                                  real *__restrict__ m)
{
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    int sel[6], na = 0;
    for (int k = 0; k < 6; k++)
        if (axes_mask & (1u << k)) sel[na++] = k;
    const real *j = J + row * (6 * N);
    const bool tall = na >= N;          // Ja itself is tall (or square): orthogonalise its N columns
    const int p = tall ? na : N, d = tall ? N : na;
    real W[10 * 6];                     // W[r * d + c], p x d
    for (int r = 0; r < p; r++)
        for (int c = 0; c < d; c++) W[r * d + c] = tall ? j[sel[r] * N + c] : j[sel[c] * N + r];
    const real eps = sizeof(real) == 8 ? (real)1e-15 : (real)1e-6;
    for (int sweep = 0; sweep < 30; sweep++) {
        bool rotated = false;
        for (int a = 0; a < d - 1; a++)
            for (int b = a + 1; b < d; b++) {
                real al = 0, be = 0, ga = 0;
                for (int r = 0; r < p; r++) {
                    const real x = W[r * d + a], y = W[r * d + b];
                    al = fma(x, x, al); be = fma(y, y, be); ga = fma(x, y, ga);
                }
                if (fabs(ga) <= eps * sqrt(al * be) || ga == 0) continue;
                rotated = true;
                const real zeta = (be - al) / (2 * ga);
                const real t = (zeta >= 0 ? (real)1 : (real)-1) / (fabs(zeta) + sqrt(1 + zeta * zeta));
                const real cs = 1 / sqrt(1 + t * t), sn = cs * t;
                for (int r = 0; r < p; r++) {
                    const real x = W[r * d + a], y = W[r * d + b];
                    W[r * d + a] = cs * x - sn * y;
                    W[r * d + b] = sn * x + cs * y;
                }
            }
        if (!rotated) break;
    }
    real smin = 0, smax = 0;
    for (int c = 0; c < d; c++) {
        real nn = 0;
        for (int r = 0; r < p; r++) nn = fma(W[r * d + c], W[r * d + c], nn);
        nn = sqrt(nn);
        if (c == 0 || nn < smin) smin = nn;
        if (c == 0 || nn > smax) smax = nn;
    }
    m[row] = kind == 0 ? smin : (smax > 0 ? smin / smax : (real)0);
}

// B2K_HESSIAN_LUT=1 keeps every call on the warp-per-row kernel (measurement / tests of that path)
static bool hessian_lut_only()
{
    static const bool v = [] { const char *e = getenv("B2K_HESSIAN_LUT"); return e && atoi(e) != 0; }();
    return v;
}

template <typename real>
static int extra_launch(int what, int n, const void *J, long long N, unsigned axes_mask, void *out, cudaStream_t st,
                        const void *aux = nullptr)
{
#define B2K_CASE(NN)                                                                                                  \
    case NN:                                                                                                          \
        if (what == 0 || what == 2) {                                                                                 \
            long long blocks = (N + 7) / 8;                                                                           \
            /* k_hessian: 4 resident blocks per SM (64 registers x 256 threads); one wave, so that the per-thread  */ \
            /* index table is set up once per ~200 rows                                                             */ \
            const long long cap = (long long)b2k_num_sms() * (what == 0 ? 4 : 16);                                    \
            if (blocks > cap) blocks = cap;                                                                           \
            if (what == 0 && NN >= 3 && ((uintptr_t)out & 15) == 0 && !hessian_lut_only() &&                          \
                b2k_blocks_per_sm((const void *)k_hessian_tile<real, NN>, 128, HessTile<real, NN>::SMEM) >= 1)         \
                k_hessian_tile<real, NN><<<(unsigned)((N + 31) / 32), 128, HessTile<real, NN>::SMEM, st>>>((const real *)J, N, (real *)out); \
            else if (what == 0) k_hessian<real, NN><<<(unsigned)blocks, 256, 0, st>>>((const real *)J, N, (real *)out, (int)(((uintptr_t)out & (2 * sizeof(real) - 1)) == 0)); \
            else k_jacob_dot_lane<real, NN><<<(unsigned)((N + B2K_XT - 1) / B2K_XT), B2K_XT, 0, st>>>((const real *)J, (const real *)aux, N, (real *)out); \
        } else if (what == 3) {                                                                                       \
            if (axes_mask == 63u && NN >= 6) k_jacobm_all<real, NN><<<(unsigned)((N + 127) / 128), 128, 0, st>>>((const real *)J, N, (real *)out); \
            else k_jacobm<real, NN><<<(unsigned)((N + 127) / 128), 128, 0, st>>>((const real *)J, N, axes_mask, (real *)out); \
        } else if (what == 4 || what == 5) {                                                                          \
            if (axes_mask == 63u) k_singular_all<real, NN><<<(unsigned)((N + 127) / 128), 128, 0, st>>>((const real *)J, N, what - 4, (real *)out); \
            else k_singular<real, NN><<<(unsigned)((N + 127) / 128), 128, 0, st>>>((const real *)J, N, axes_mask, what - 4, (real *)out); \
        } else if (axes_mask == 63u && NN > 6) {                                                                      \
            k_yoshikawa_all<real, NN><<<(unsigned)((N + B2K_XT - 1) / B2K_XT), B2K_XT, 0, st>>>((const real *)J, N, (real *)out); \
        } else {                                                                                                      \
            k_yoshikawa<real, NN><<<(unsigned)((N + 127) / 128), 128, 0, st>>>((const real *)J, N, axes_mask, (real *)out); \
        }                                                                                                             \
        break;
    switch (n) {
        B2K_CASE(1) B2K_CASE(2) B2K_CASE(3) B2K_CASE(4) B2K_CASE(5)
        B2K_CASE(6) B2K_CASE(7) B2K_CASE(8) B2K_CASE(9) B2K_CASE(10)
    default:
        b2k_set_error("unsupported joint count %d", n);
        return B2K_ERR_INVALID;
    }
#undef B2K_CASE
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

extern "C" int b2k_hessian(int dtype, int n, const void *J, int64_t N, void *H, void *stream)
{
    if (N < 0 || (N > 0 && (!J || !H))) { b2k_set_error("b2k_hessian: bad arguments"); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("b2k_hessian: bad dtype"); return B2K_ERR_INVALID; }
    if (n < 1 || n > B2K_MAX_JOINTS) { b2k_set_error("b2k_hessian: unsupported joint count %d", n); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(J);
    return dtype == B2K_F64 ? extra_launch<double>(0, n, J, N, 0, H, (cudaStream_t)stream)
                            : extra_launch<float>(0, n, J, N, 0, H, (cudaStream_t)stream);
}

extern "C" int b2k_manipulability(int dtype, int n, const void *J, int64_t N, uint32_t axes_mask, void *m, void *stream)
{
    if (N < 0 || (N > 0 && (!J || !m))) { b2k_set_error("b2k_manipulability: bad arguments"); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("b2k_manipulability: bad dtype"); return B2K_ERR_INVALID; }
    if (n < 1 || n > B2K_MAX_JOINTS) { b2k_set_error("b2k_manipulability: unsupported joint count %d", n); return B2K_ERR_INVALID; }
    if ((axes_mask & 63u) == 0) { b2k_set_error("b2k_manipulability: no Cartesian axis selected"); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(J);
    return dtype == B2K_F64 ? extra_launch<double>(1, n, J, N, axes_mask & 63u, m, (cudaStream_t)stream)
                            : extra_launch<float>(1, n, J, N, axes_mask & 63u, m, (cudaStream_t)stream);
}


extern "C" int b2k_manipulability_svd(int dtype, int n, const void *J, int64_t N, uint32_t axes_mask, int kind, void *m, void *stream)
{
    if (N < 0 || (N > 0 && (!J || !m))) { b2k_set_error("b2k_manipulability_svd: bad arguments"); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("b2k_manipulability_svd: bad dtype"); return B2K_ERR_INVALID; }
    if (n < 1 || n > B2K_MAX_JOINTS) { b2k_set_error("b2k_manipulability_svd: unsupported joint count %d", n); return B2K_ERR_INVALID; }
    if ((axes_mask & 63u) == 0) { b2k_set_error("b2k_manipulability_svd: no Cartesian axis selected"); return B2K_ERR_INVALID; }
    if (kind != 0 && kind != 1) { b2k_set_error("b2k_manipulability_svd: kind must be 0 (minsingular) or 1 (invcondition)"); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(J);
    return dtype == B2K_F64 ? extra_launch<double>(4 + kind, n, J, N, axes_mask & 63u, m, (cudaStream_t)stream)
                            : extra_launch<float>(4 + kind, n, J, N, axes_mask & 63u, m, (cudaStream_t)stream);
}

extern "C" int b2k_jacob_dot(int dtype, int n, const void *J, const void *qd, int64_t N, void *Jd, void *stream)
{
    if (N < 0 || (N > 0 && (!J || !qd || !Jd))) { b2k_set_error("b2k_jacob_dot: bad arguments"); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("b2k_jacob_dot: bad dtype"); return B2K_ERR_INVALID; }
    if (n < 1 || n > B2K_MAX_JOINTS) { b2k_set_error("b2k_jacob_dot: unsupported joint count %d", n); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(J);
    return dtype == B2K_F64 ? extra_launch<double>(2, n, J, N, 0, Jd, (cudaStream_t)stream, qd)
                            : extra_launch<float>(2, n, J, N, 0, Jd, (cudaStream_t)stream, qd);
}

extern "C" int b2k_jacobm(int dtype, int n, const void *J, int64_t N, uint32_t axes_mask, void *Jm, void *stream)
{
    if (N < 0 || (N > 0 && (!J || !Jm))) { b2k_set_error("b2k_jacobm: bad arguments"); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("b2k_jacobm: bad dtype"); return B2K_ERR_INVALID; }
    if (n < 1 || n > B2K_MAX_JOINTS) { b2k_set_error("b2k_jacobm: unsupported joint count %d", n); return B2K_ERR_INVALID; }
    if ((axes_mask & 63u) == 0) { b2k_set_error("b2k_jacobm: no Cartesian axis selected"); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(J);
    return dtype == B2K_F64 ? extra_launch<double>(3, n, J, N, axes_mask & 63u, Jm, (cudaStream_t)stream)
                            : extra_launch<float>(3, n, J, N, axes_mask & 63u, Jm, (cudaStream_t)stream);
}


// ------------------------------------------------------------------ joint-space trajectory producer (SURVEY 8f-3)
// jtraj (reference tools/trajectory.py:686-780): quintic blend q0 -> qf with boundary velocities qd0, qd1:
//   q(s) = A s^5 + B s^4 + C s^3 + E s + F,  qd = (5A s^4 + 4B s^3 + 3C s^2 + E) / tscal,
//   qdd = (20A s^3 + 12B s^2 + 6C s) / tscal^2,  s = t / tscal in [0, 1].
// Rows are time samples; one thread per (row, joint) element so the three (N,n) outputs are written coalesced and a
// q batch is produced where the FK / RNE kernels consume it, without a host round trip.
struct JtrajP {
    double A[B2K_MAX_JOINTS], B[B2K_MAX_JOINTS], C[B2K_MAX_JOINTS], E[B2K_MAX_JOINTS], F[B2K_MAX_JOINTS];
    double inv_tscal, inv_nm1;
    int n;
};

template <typename real>
__global__ void __launch_bounds__(256) k_jtraj(const __grid_constant__ JtrajP P, const real *__restrict__ ts, long long nrows,
                                               real *__restrict__ q, real *__restrict__ qd, real *__restrict__ qdd)
{
    const long long total = nrows * P.n;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        long long row; int j;
        split_elem(e, P.n, total, row, j);
        // normalised time: the caller's samples, or np.linspace(0, 1, N)[row] (last sample exactly 1)
        const real s = ts ? ts[row] * (real)P.inv_tscal
                          : (row == nrows - 1 ? (real)1 : (real)((double)row * P.inv_nm1));
        const real A = (real)P.A[j], B = (real)P.B[j], C = (real)P.C[j], E = (real)P.E[j], F = (real)P.F[j];
        const real it = (real)P.inv_tscal;
        q[e] = fma(fma(fma(fma(A, s, B), s, C) * s, s, E), s, F);
        if (qd) qd[e] = fma(fma(fma((real)5 * A, s, (real)4 * B), s, (real)3 * C) * s, s, E) * it;
        if (qdd) qdd[e] = fma(fma((real)20 * A, s, (real)12 * B), s, (real)6 * C) * s * it * it;
    }
}

extern "C" int b2k_jtraj(int dtype, int n, const double *q0, const double *qf, const double *qd0, const double *qd1,
                         int64_t N, const void *t, double tscal, void *q, void *qd, void *qdd, void *stream)
{
    const char *fn = "b2k_jtraj";
    if (n < 1 || n > B2K_MAX_JOINTS) { b2k_set_error("%s: n must be 1..%d", fn, B2K_MAX_JOINTS); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (!q0 || !qf) { b2k_set_error("%s: q0 / qf is NULL", fn); return B2K_ERR_INVALID; }
    if (N < 0 || (N > 0 && !q)) { b2k_set_error("%s: bad N / q", fn); return B2K_ERR_INVALID; }
    if (!(tscal > 0)) { b2k_set_error("%s: tscal must be positive", fn); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(q);
    JtrajP P;
    P.n = n;
    P.inv_tscal = 1.0 / tscal;
    P.inv_nm1 = N > 1 ? 1.0 / (double)(N - 1) : 0.0;
    for (int j = 0; j < n; j++) { // trajectory.py:753-757
        const double d = qf[j] - q0[j], v0 = qd0 ? qd0[j] : 0.0, v1 = qd1 ? qd1[j] : 0.0;
        P.A[j] = 6 * d - 3 * (v1 + v0) * tscal;
        P.B[j] = -15 * d + (8 * v0 + 7 * v1) * tscal;
        P.C[j] = 10 * d - (6 * v0 + 4 * v1) * tscal;
        P.E[j] = v0 * tscal;
        P.F[j] = q0[j];
    }
    const long long total = N * n;
    long long blocks = (total + 255) / 256;
    const long long cap = (long long)b2k_num_sms() * 16;
    if (blocks > cap) blocks = cap;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == B2K_F64)
        k_jtraj<double><<<(unsigned)blocks, 256, 0, st>>>(P, (const double *)t, N, (double *)q, (double *)qd, (double *)qdd);
    else
        k_jtraj<float><<<(unsigned)blocks, 256, 0, st>>>(P, (const float *)t, N, (float *)q, (float *)qd, (float *)qdd);
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}


// ------------------------------------------------------------------ pose error / position-based servo
// Batched fknm.Angle_Axis (fknm.cpp:112-162 -> _angle_axis ik.cpp:241-286) and tools/p_servo.py:46-106 with
// method="angle-axis": e = angle_axis(Te, Tep), v = gain .* e, arrived = sum|e| < threshold.
// Lane per row; tep_stride = 0 broadcasts one target to every row.
template <typename real, bool VEC>
__global__ void __launch_bounds__(256) k_pose_error(const real *__restrict__ Te, const real *__restrict__ Tep,
                                                    long long tep_stride, long long nrows, real g0, real g1, real g2,
                                                    real g3, real g4, real g5, real threshold, real *__restrict__ out,
                                                    int *__restrict__ arrived)
{
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    // the three used rows of each 4x4 matrix as 16-byte vector loads where both arrays are 16-byte aligned (the launcher
    // looks; any torch allocation is): a third of the load instructions of the scalar form
    real ar[12], Tp[12], e[6];
    if (VEC) {
        load12<real>(Te + row * 16, ar);
        load12<real>(Tep + row * tep_stride, Tp);
    } else {
#pragma unroll
        for (int k = 0; k < 12; k++) { ar[k] = Te[row * 16 + k]; Tp[k] = Tep[row * tep_stride + k]; }
    }
    Pose<real> T;
    pose_from_const<real>(T, ar);
    ik_angle_axis<real>(T, Tp, e);
    const real g[6] = {g0, g1, g2, g3, g4, g5};
    real sum = 0;
#pragma unroll
    for (int k = 0; k < 6; k++) {
        sum += fabs(e[k]);
        out[row * 6 + k] = g[k] * e[k];
    }
    if (arrived) arrived[row] = sum < threshold ? 1 : 0;
}

static int pose_error_launch(const char *fn, int dtype, const void *Te, const void *Tep, int64_t N, int64_t tep_stride,
                             const double *gain, double threshold, void *out, int32_t *arrived, void *stream)
{
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (N < 0 || (N > 0 && (!Te || !Tep || !out))) { b2k_set_error("%s: bad arguments", fn); return B2K_ERR_INVALID; }
    if (tep_stride != 0 && tep_stride != 16) { b2k_set_error("%s: tep_stride must be 0 (one target) or 16", fn); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(Te);
    double g[6];
    for (int k = 0; k < 6; k++) g[k] = gain ? gain[k] : 1.0;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)((N + 255) / 256);
    const bool vec = (((uintptr_t)Te | (uintptr_t)Tep) & 15) == 0;
#define B2K_PE(REAL, V)                                                                                                        \
    k_pose_error<REAL, V><<<blocks, 256, 0, st>>>((const REAL *)Te, (const REAL *)Tep, tep_stride, N, (REAL)g[0], (REAL)g[1], \
                                                  (REAL)g[2], (REAL)g[3], (REAL)g[4], (REAL)g[5], (REAL)threshold, (REAL *)out, arrived)
    if (dtype == B2K_F64) { if (vec) B2K_PE(double, true); else B2K_PE(double, false); }
    else { if (vec) B2K_PE(float, true); else B2K_PE(float, false); }
#undef B2K_PE
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

extern "C" int b2k_angle_axis(int dtype, const void *Te, const void *Tep, int64_t N, int64_t tep_stride, void *e, void *stream)
{
    return pose_error_launch("b2k_angle_axis", dtype, Te, Tep, N, tep_stride, nullptr, 0.0, e, nullptr, stream);
}

extern "C" int b2k_p_servo(int dtype, const void *Te, const void *Tep, int64_t N, int64_t tep_stride, const double *gain,
                           double threshold, void *v, int32_t *arrived, void *stream)
{
    if (N > 0 && !arrived) { b2k_set_error("b2k_p_servo: arrived is NULL"); return B2K_ERR_INVALID; }
    return pose_error_launch("b2k_p_servo", dtype, Te, Tep, N, tep_stride, gain, threshold, v, arrived, stream);
}

// ------------------------------------------------------------------ scalar / multi-axis trajectory profiles (SURVEY 8f-3)
// quintic (tools/trajectory.py:271-416), trapezoidal (429-615) and their multi-axis form mtraj (617-684): every axis
// follows the same kind of profile between its own end points.  The per-axis parameters are worked out on the host in
// fp64 (quintic: the 6x6 boundary-condition system of quintic_func; trapezoidal: V, blend time tb and acceleration a of
// trapezoidal_func); one thread per (sample, axis) element evaluates position, velocity and acceleration.
struct MtrajP {
    double c[B2K_MAX_JOINTS][6]; // quintic: polynomial coefficients, highest power first; trapezoidal: q0, qf, V, tb, a, T
    int n, kind;
};

template <typename real>
__global__ void __launch_bounds__(256) k_mtraj(const __grid_constant__ MtrajP P, const real *__restrict__ t, long long nrows,
                                               real *__restrict__ s, real *__restrict__ sd, real *__restrict__ sdd)
{
    const long long total = nrows * P.n;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        long long row; int j;
        split_elem(e, P.n, total, row, j);
        const real tk = t ? t[row] : (real)row; // `t: int` means t = arange(0, t) (trajectory.py:330, 489)
        real p, pd, pdd;
        if (P.kind == 0) { // np.polyval of coeffs, coeffs_d, coeffs_dd (trajectory.py:405-415)
            const real c5 = (real)P.c[j][0], c4 = (real)P.c[j][1], c3 = (real)P.c[j][2], c2 = (real)P.c[j][3],
                       c1 = (real)P.c[j][4], c0 = (real)P.c[j][5];
            p = fma(fma(fma(fma(fma(c5, tk, c4), tk, c3), tk, c2), tk, c1), tk, c0);
            pd = fma(fma(fma(fma((real)5 * c5, tk, (real)4 * c4), tk, (real)3 * c3), tk, (real)2 * c2), tk, c1);
            pdd = fma(fma(fma((real)20 * c5, tk, (real)12 * c4), tk, (real)6 * c3), tk, (real)2 * c2);
        } else { // trapezoidalfunc (trajectory.py:566-600)
            const real q0 = (real)P.c[j][0], qf = (real)P.c[j][1], V = (real)P.c[j][2], tb = (real)P.c[j][3],
                       a = (real)P.c[j][4], T = (real)P.c[j][5];
            if (tk < 0) { p = q0; pd = 0; pdd = 0; }
            else if (tk <= tb) { p = q0 + a / 2 * tk * tk; pd = a * tk; pdd = a; }
            else if (tk <= T - tb) { p = (qf + q0 - V * T) / 2 + V * tk; pd = V; pdd = 0; }
            else if (tk <= T) { p = qf - a / 2 * T * T + a * T * tk - a / 2 * tk * tk; pd = a * T - a * tk; pdd = -a; }
            else { p = qf; pd = 0; pdd = 0; }
        }
        s[e] = p;
        if (sd) sd[e] = pd;
        if (sdd) sdd[e] = pdd;
    }
}

// solve the 6x6 system of quintic_func (Gaussian elimination with partial pivoting, fp64)
static bool quintic_coeffs(double q0, double qf, double T, double v0, double vf, double *c)
{
    const double T2 = T * T, T3 = T2 * T, T4 = T3 * T, T5 = T4 * T;
    double X[6][7] = {{0, 0, 0, 0, 0, 1, q0},          {T5, T4, T3, T2, T, 1, qf},         {0, 0, 0, 0, 1, 0, v0},
                      {5 * T4, 4 * T3, 3 * T2, 2 * T, 1, 0, vf}, {0, 0, 0, 2, 0, 0, 0}, {20 * T3, 12 * T2, 6 * T, 2, 0, 0, 0}};
    for (int k = 0; k < 6; k++) {
        int p = k;
        for (int i = k + 1; i < 6; i++)
            if (fabs(X[i][k]) > fabs(X[p][k])) p = i;
        if (X[p][k] == 0.0) return false;
        if (p != k)
            for (int j = 0; j < 7; j++) { double tmp = X[k][j]; X[k][j] = X[p][j]; X[p][j] = tmp; }
        for (int i = k + 1; i < 6; i++) {
            const double f = X[i][k] / X[k][k];
            for (int j = k; j < 7; j++) X[i][j] -= f * X[k][j];
        }
    }
    for (int i = 5; i >= 0; i--) {
        double acc = X[i][6];
        for (int j = i + 1; j < 6; j++) acc -= X[i][j] * c[j];
        c[i] = acc / X[i][i];
    }
    return true;
}

extern "C" int b2k_mtraj(int dtype, int kind, int n, const double *q0, const double *qf, const double *qd0, const double *qdf,
                         const double *V, int64_t N, const void *t, double tf, void *s, void *sd, void *sdd, double *tblend,
                         void *stream)
{
    const char *fn = "b2k_mtraj";
    if (n < 1 || n > B2K_MAX_JOINTS) { b2k_set_error("%s: n must be 1..%d", fn, B2K_MAX_JOINTS); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (kind != 0 && kind != 1) { b2k_set_error("%s: kind must be 0 (quintic) or 1 (trapezoidal)", fn); return B2K_ERR_INVALID; }
    if (!q0 || !qf) { b2k_set_error("%s: q0 / qf is NULL", fn); return B2K_ERR_INVALID; }
    if (N < 0 || (N > 0 && !s)) { b2k_set_error("%s: bad N / output", fn); return B2K_ERR_INVALID; }
    if (!(tf > 0)) { b2k_set_error("%s: the final time must be positive (at least two samples)", fn); return B2K_ERR_INVALID; }
    MtrajP P;
    P.n = n;
    P.kind = kind;
    for (int j = 0; j < n; j++) {
        if (kind == 0) {
            if (!quintic_coeffs(q0[j], qf[j], tf, qd0 ? qd0[j] : 0.0, qdf ? qdf[j] : 0.0, P.c[j])) {
                b2k_set_error("%s: singular boundary-condition system", fn);
                return B2K_ERR_INVALID;
            }
        } else { // trapezoidal_func, trajectory.py:552-565
            double v;
            if (!V || V[j] != V[j]) v = (qf[j] - q0[j]) / tf * 1.5; // NaN = not given
            else {
                const double d = qf[j] - q0[j];
                v = fabs(V[j]) * (d > 0 ? 1.0 : (d < 0 ? -1.0 : 0.0));
                if (fabs(v) < fabs(d) / tf) { b2k_set_error("V too small"); return B2K_ERR_INVALID; }
                if (fabs(v) > 2 * fabs(d) / tf) { b2k_set_error("V too big"); return B2K_ERR_INVALID; }
            }
            double tb, a;
            if (v == 0) { tb = INFINITY; a = 0; }
            else { tb = (q0[j] - qf[j] + v * tf) / v; a = v / tb; }
            P.c[j][0] = q0[j]; P.c[j][1] = qf[j]; P.c[j][2] = v; P.c[j][3] = tb; P.c[j][4] = a; P.c[j][5] = tf;
            if (tblend) tblend[j] = tb;
        }
    }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(s);
    const long long total = N * n;
    long long blocks = (total + 255) / 256;
    const long long cap = (long long)b2k_num_sms() * 16;
    if (blocks > cap) blocks = cap;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == B2K_F64)
        k_mtraj<double><<<(unsigned)blocks, 256, 0, st>>>(P, (const double *)t, N, (double *)s, (double *)sd, (double *)sdd);
    else
        k_mtraj<float><<<(unsigned)blocks, 256, 0, st>>>(P, (const float *)t, N, (float *)s, (float *)sd, (float *)sdd);
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}
