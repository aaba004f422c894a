// b2k_fkw.cu -- measurement variant 1: the literal "one warp = one joint configuration" walk.
//
// BASELINE.json's north_star describes the kernel as one warp per configuration.  This file
// implements exactly that so the choice can be measured instead of argued (DESIGN.md "Why a
// lane per configuration"): the 3x4 pose lives one element per lane (lanes 0..11), every chain
// step is a handful of __shfl_sync + FMA on those 12 lanes, the n sincos are evaluated by n lanes
// in parallel, the Jacobian columns are formed by 3n lanes, outputs are written coalesced by the
// warp.  20 of 32 lanes idle through the serial part, and every instruction serves ONE row
// instead of 32: measured several times slower than the default kernel.
// Supported for "DH-like" chains only (unflipped Rz joints, any constants): it is a measurement
// aid selected with b2k_set_variant(1), not a product path.
#include "b2k_fkj.cuh"

template <typename real, int N>
struct FkwP {
    real A[N + 1][12];
    real B[12];
    int has_base;
    int jidx[N];
    TrigC<real> trig;
};

template <typename real, int N, bool WT, bool WJ>
__global__ void __launch_bounds__(256)
k_fkw(const __grid_constant__ FkwP<real, N> P, const real *__restrict__ q, long long nrows, int ldq,
      real *__restrict__ Tout, real *__restrict__ Jout)
{
    __shared__ real sA[(N + 1) * 12 + 12];
    __shared__ real sZP[8][N][6]; // per warp: z_j (3) | p_j (3)
    for (int i = threadIdx.x; i < (N + 1) * 12; i += blockDim.x) sA[i] = P.A[i / 12][i % 12];
    for (int i = threadIdx.x; i < 12; i += blockDim.x) sA[(N + 1) * 12 + i] = P.B[i];
    __syncthreads();
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int r = (lane >> 2) % 3, c = lane & 3; // pose element owned by lanes 0..11
    const long long wstride = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + warp; row < nrows; row += wstride) {
        // n lanes evaluate the n sincos in parallel
        real s = 0, cs = 1;
        if (lane < N) b2k_sincos(q[row * ldq + P.jidx[lane]], P.trig, &s, &cs);
        real t = sA[r * 4 + c]; // T = A_0
#pragma unroll
        for (int j = 0; j < N; j++) {
            if (j > 0) { // T <- T * A_j : element (r,c) = sum_k T(r,k) A_j(k,c) (+ T(r,3) for c == 3)
                const real *A = sA + j * 12;
                const real t0 = __shfl_sync(FULL, t, (lane & ~3) | 0), t1 = __shfl_sync(FULL, t, (lane & ~3) | 1);
                const real t2 = __shfl_sync(FULL, t, (lane & ~3) | 2), t3 = __shfl_sync(FULL, t, (lane & ~3) | 3);
                t = fma(t0, A[0 * 4 + c], fma(t1, A[1 * 4 + c], t2 * A[2 * 4 + c])) + (c == 3 ? t3 : (real)0);
            }
            if (WJ && lane < 12 && c >= 2) sZP[warp][j][(c - 2) * 3 + r] = t; // column 2 = z_j, column 3 = p_j
            // T <- T * Rz(q_j): columns 0 and 1 mix
            const real sj = __shfl_sync(FULL, s, j), cj = __shfl_sync(FULL, cs, j);
            const real other = __shfl_xor_sync(FULL, t, 1);
            if (c == 0) t = fma(cj, t, sj * other);
            else if (c == 1) t = fma(cj, t, -(sj * other));
        }
        { // tail constant
            const real *A = sA + N * 12;
            const real t0 = __shfl_sync(FULL, t, (lane & ~3) | 0), t1 = __shfl_sync(FULL, t, (lane & ~3) | 1);
            const real t2 = __shfl_sync(FULL, t, (lane & ~3) | 2), t3 = __shfl_sync(FULL, t, (lane & ~3) | 3);
            t = fma(t0, A[0 * 4 + c], fma(t1, A[1 * 4 + c], t2 * A[2 * 4 + c])) + (c == 3 ? t3 : (real)0);
        }
        if (WJ) {
            __syncwarp();
            // p_e components live in lanes 3, 7, 11
            const real pex = __shfl_sync(FULL, t, 3), pey = __shfl_sync(FULL, t, 7), pez = __shfl_sync(FULL, t, 11);
            for (int e = lane; e < 6 * N; e += 32) { // element e = k * N + j of the 6 x N Jacobian
                const int k = e / N, j = e - k * N;
                const real *zp = sZP[warp][j];
                real v;
                if (k >= 3) v = zp[k - 3];
                else {
                    const real dx = pex - zp[3], dy = pey - zp[4], dz = pez - zp[5];
                    v = (k == 0) ? fma(zp[1], dz, -(zp[2] * dy)) : (k == 1) ? fma(zp[2], dx, -(zp[0] * dz)) : fma(zp[0], dy, -(zp[1] * dx));
                }
                Jout[row * (6 * N) + e] = v;
            }
            __syncwarp();
        }
        if (WT) {
            real v = t;
            if (P.has_base) { // T <- B * T : element (r,c) = sum_k B(r,k) T(k,c) (+ B(r,3) for c == 3)
                const real *Bm = sA + (N + 1) * 12;
                const real u0 = __shfl_sync(FULL, t, c), u1 = __shfl_sync(FULL, t, 4 + c), u2 = __shfl_sync(FULL, t, 8 + c);
                v = fma(Bm[r * 4 + 0], u0, fma(Bm[r * 4 + 1], u1, Bm[r * 4 + 2] * u2)) + (c == 3 ? Bm[r * 4 + 3] : (real)0);
            }
            if (lane < 12) Tout[row * 16 + lane] = v;
            else if (lane < 16) Tout[row * 16 + lane] = (lane == 15) ? (real)1 : (real)0;
        }
    }
}

template <typename real, int N>
static int fkw_launch_n(const b2k_chain_s *c, int mode, const real *q, long long nrows, int ldq, const double *base,
                        const double *tool, real *T, real *J, cudaStream_t st)
{
    ChainP<real, N> C;
    const bool wt = mode & FKJ_T, wj = mode & FKJ_J0;
    b2k_fill_chain<real, N>(c, base, tool, wt && !wj, C);
    FkwP<real, N> P;
    for (int j = 0; j <= N; j++)
        for (int k = 0; k < 12; k++) P.A[j][k] = C.A[j][k];
    for (int k = 0; k < 12; k++) P.B[k] = C.B[k];
    P.has_base = C.has_base;
    for (int j = 0; j < N; j++) P.jidx[j] = C.jidx[j];
    P.trig = C.trig;
    long long blocks = (nrows + 7) / 8;
    const long long cap = (long long)b2k_num_sms() * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    if (wt && wj) k_fkw<real, N, true, true><<<(unsigned)blocks, 256, 0, st>>>(P, q, nrows, ldq, T, J);
    else if (wt) k_fkw<real, N, true, false><<<(unsigned)blocks, 256, 0, st>>>(P, q, nrows, ldq, T, J);
    else k_fkw<real, N, false, true><<<(unsigned)blocks, 256, 0, st>>>(P, q, nrows, ldq, T, J);
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

int b2k_fkw_launch(const b2k_chain_s *c, int dtype, int mode, const void *q, long long nrows, long long ldq,
                   const double *base, const double *tool, void *T, void *J, cudaStream_t st)
{
    if (!c->all_rz) {
        b2k_set_error("variant 1 (warp per configuration) is a measurement aid for chains of unflipped Rz joints only");
        return B2K_ERR_INVALID;
    }
#define B2K_CASE(NN)                                                                                                        \
    case NN:                                                                                                                \
        return dtype == B2K_F64                                                                                             \
                   ? fkw_launch_n<double, NN>(c, mode, (const double *)q, nrows, (int)ldq, base, tool, (double *)T, (double *)J, st) \
                   : fkw_launch_n<float, NN>(c, mode, (const float *)q, nrows, (int)ldq, base, tool, (float *)T, (float *)J, st);
    switch (c->n) {
        B2K_CASE(6) B2K_CASE(7)
    default:
        b2k_set_error("variant 1 is built for n = 6 and n = 7 only");
        return B2K_ERR_INVALID;
    }
#undef B2K_CASE
}
