// b2k_ik6s.cu -- closed-form inverse kinematics of a Puma-type 6R arm: the reference's DHRobot.ikine_6s (Puma560.ikine_a)
// over a batch of poses, every requested shoulder / elbow / wrist configuration from one read of each pose.
//
// One lane per row, 64-thread blocks.  Each warp stages its 32 poses through shared memory with 16-byte loads (odd row
// pitch, so the lanes then read their own rows without bank conflicts), and the same stage then collects the (nconf, 6)
// joint rows and the ok flags so that they leave coalesced.  Per row the wrist centre W = base^-1 T tool^-1 Tt^-1, its
// distance r from the first axis and atan2(Py, Px) are formed once; per shoulder theta1, V, the elbow cosine and
// Rz(theta1)^T R(W); per configuration the rest.  With the pattern's twists R(A1 A2 A3) = Rz(theta1) Ry(-(theta2 +
// theta3)), so R(A1 A2 A3)^T R(W) is two plane rotations of R(W), not three link products.  DESIGN (f-6) states the
// algorithm and what the configuration letters mean.
#include <math.h>

#include "b2k_common.cuh"

#define B2K_IK6_WARPS 2

namespace {

template <typename real>
struct Ik6sP {
    real Bi[12];   // base^-1, 3x4 row-major
    real Ei[12];   // tool^-1 Tt^-1, Tt = transl(a6, 0, d6) Rx(alpha6)
    real d1, D;    // D = d2 + d3
    real a2, k2, two_a2, beta3; // k2 = a2^2 - a3^2 - d4^2, beta3 = atan2(a3, d4)
    real sign_a2;
    real off[6];
    int wrist_neg; // alpha4 > 0: theta5 is the negated tr2eul theta
    int conf[8];
    int vec;       // T is 16-byte aligned
    long long nrows;
};

// C = A B for affine 3x4 matrices
template <typename real>
__device__ __forceinline__ void ik6_mul34(const real *A, const real *B, real *C)
{
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
        for (int j = 0; j < 4; j++) {
            real s = j == 3 ? A[i * 4 + 3] : (real)0;
#pragma unroll
            for (int k = 0; k < 3; k++) s = fma(A[i * 4 + k], B[k * 4 + j], s);
            C[i * 4 + j] = s;
        }
    }
}

// (x + pi) mod 2pi - pi with numpy's floor modulo: the remainder a - k 2pi is exact, so one fma gives it
template <typename real>
__device__ __forceinline__ real ik6_wrap(real x)
{
    const real pi = (real)3.14159265358979323846, tau = (real)6.283185307179586;
    const real a = x + pi;
    const real k = floor(a * ((real)1 / tau));
    real w = fma(-k, tau, a);
    if (w < 0) w += tau;
    else if (w >= tau) w -= tau;
    return w - pi;
}

// sin and cos of the angles this kernel forms, all below 8 pi in magnitude (or NaN on a row that is out of reach):
// sincospi needs no Payne-Hanek reduction, whose local array would give the kernel a stack frame
struct Ik6SinCos {
    __device__ __forceinline__ void operator()(double x, double &s, double &c) const { sincospi(x * 0.31830988618379067, &s, &c); }
    __device__ __forceinline__ void operator()(float x, float &s, float &c) const { sincospif(x * 0.31830988618f, &s, &c); }
};

template <typename real> __device__ __forceinline__ void ik6_ld16(const real *p, real *o);
template <> __device__ __forceinline__ void ik6_ld16<double>(const double *p, double *o)
{
    const double2 v = __ldg(reinterpret_cast<const double2 *>(p));
    o[0] = v.x; o[1] = v.y;
}
template <> __device__ __forceinline__ void ik6_ld16<float>(const float *p, float *o)
{
    const float4 v = __ldg(reinterpret_cast<const float4 *>(p));
    o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
}

template <typename real, int NC>
__global__ void __launch_bounds__(32 * B2K_IK6_WARPS) k_ikine_6s(const __grid_constant__ Ik6sP<real> P, const real *__restrict__ T,
                                                                  real *__restrict__ q, int *__restrict__ ok)
{
    constexpr int TS = 17;                  // odd pitch of a staged pose row
    constexpr int QW = 6 * NC, QS = QW + 1; // a row of q, and its odd pitch in the stage
    constexpr int OS = NC | 1;              // odd pitch of a row of ok flags
    constexpr int SS = TS > QS ? TS : QS;
    __shared__ real stage[B2K_IK6_WARPS][32 * SS];
    __shared__ int okst[B2K_IK6_WARPS][32 * OS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long row0 = ((long long)blockIdx.x * B2K_IK6_WARPS + warp) * 32;
    if (row0 >= P.nrows) return;
    const int rows = (int)(P.nrows - row0 < 32 ? P.nrows - row0 : 32);
    real *st = stage[warp];
    int *so = okst[warp];

    const real *src = T + row0 * 16;
    if (P.vec) {
        constexpr int U = 16 / sizeof(real), UPR = 16 / U; // reals per 16-byte unit, units per pose
        for (int u = lane; u < rows * UPR; u += 32) {
            real v[U];
            ik6_ld16<real>(src + u * U, v);
            const int r = u / UPR, c = (u % UPR) * U;
#pragma unroll
            for (int j = 0; j < U; j++) st[r * TS + c + j] = v[j];
        }
    } else {
        for (int e = lane; e < rows * 16; e += 32) st[(e >> 4) * TS + (e & 15)] = src[e];
    }
    __syncwarp();
    const int lr = lane < rows ? lane : 0; // idle lanes of a ragged tile recompute row 0 and store nothing
    real t[12], M[12], W[12];
#pragma unroll
    for (int k = 0; k < 12; k++) t[k] = st[lr * TS + k];
    __syncwarp(); // the stage now collects the output

    // wrist centre and the quantities every configuration shares
    ik6_mul34<real>(P.Bi, t, M);
    ik6_mul34<real>(M, P.Ei, W);
    const real pi = (real)3.14159265358979323846;
    const Ik6SinCos sc;
    const real Px = W[3], Py = W[7], Z = W[11] - P.d1;
    const real r = hypot(Px, Py);
    const bool reach = fabs(P.D) <= r;
    const real phi = r_atan2<real>(Py, Px), s = asin(P.D / r);
    // per shoulder (index 0 = l, 1 = r): theta1, V, atan2(Z, V), acos of the elbow cosine, Rz(theta1)^T R(W) rows 0 and 1
    real th1[2], V[2], base2[2], ac[2], m0[2][3], m1[2][3];
    bool elbow_ok[2];
#pragma unroll
    for (int sh = 0; sh < 2; sh++) {
        th1[sh] = phi + (sh ? s : pi - s);
        real s1, c1;
        sc(th1[sh], s1, c1);
        V[sh] = Px * c1 + Py * s1;
        const real rho2 = V[sh] * V[sh] + Z * Z;
        const real c = (P.k2 + rho2) / (P.two_a2 * sqrt(rho2));
        elbow_ok[sh] = fabs(c) <= 1; // false for NaN and infinity too
        ac[sh] = P.sign_a2 * acos(c); // so that "u" is the elbow above the shoulder-wrist line for either sign of a2
        base2[sh] = r_atan2<real>(Z, V[sh]);
#pragma unroll
        for (int j = 0; j < 3; j++) {
            m0[sh][j] = c1 * W[j] + s1 * W[4 + j];
            m1[sh][j] = c1 * W[4 + j] - s1 * W[j];
        }
    }

#pragma unroll 1
    for (int k = 0; k < NC; k++) {
        const int code = P.conf[k];
        const bool right = code & 1, down = code & 2, flip = code & 4;
        // ternaries, not a run-time index, keep the per-shoulder values in registers
        const real t1 = right ? th1[1] : th1[0], v = right ? V[1] : V[0];
        const real th2 = (right ? base2[1] : base2[0]) + (down != right ? (real)1 : (real)-1) * (right ? ac[1] : ac[0]);
        real s2, c2;
        sc(th2, s2, c2);
        const real num = c2 * v + s2 * Z - P.a2, den = c2 * Z - s2 * v;
        const real th3 = P.beta3 - r_atan2<real>(num, den);
        real sb, cb;
        sc(th2 + th3, sb, cb);
        // R = Ry(theta2 + theta3) Rz(theta1)^T R(W)
        real R[3][3];
#pragma unroll
        for (int j = 0; j < 3; j++) {
            const real a0 = right ? m0[1][j] : m0[0][j];
            R[0][j] = cb * a0 + sb * W[8 + j];
            R[1][j] = right ? m1[1][j] : m1[0][j];
            R[2][j] = cb * W[8 + j] - sb * a0;
        }
        real g[3];
        if (flip) rot_to_eul<real, true, Ik6SinCos>(R, g);
        else rot_to_eul<real, false, Ik6SinCos>(R, g);
        const real th[6] = {t1, th2, th3, g[0], P.wrist_neg ? -g[1] : g[1], g[2]};
        const bool good = reach && (right ? elbow_ok[1] : elbow_ok[0]);
#pragma unroll
        for (int j = 0; j < 6; j++) st[lane * QS + k * 6 + j] = good ? ik6_wrap<real>(th[j] - P.off[j]) : (real)NAN;
        so[lane * OS + k] = good;
    }
    __syncwarp();
    real *qd = q + row0 * QW;
    for (int e = lane; e < rows * QW; e += 32) {
        const int r2 = e / QW;
        qd[e] = st[r2 * QS + (e - r2 * QW)];
    }
    int *od = ok + row0 * NC;
    for (int e = lane; e < rows * NC; e += 32) {
        const int r2 = e / NC;
        od[e] = so[r2 * OS + (e - r2 * NC)];
    }
}

// inverse of a rigid 3x4 transform: [R^T | -R^T t]
void ik6_inv_rigid(const double *A, double *X)
{
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) X[i * 4 + j] = A[j * 4 + i];
        X[i * 4 + 3] = -(A[0 * 4 + i] * A[3] + A[1 * 4 + i] * A[7] + A[2 * 4 + i] * A[11]);
    }
}

template <typename real>
int ik6_launch(const double *Bi, const double *Ei, const double *dh, const void *T, long long N, int nconf, const int32_t *conf,
               void *q, int32_t *ok, cudaStream_t st)
{
    Ik6sP<real> P;
    for (int k = 0; k < 12; k++) { P.Bi[k] = (real)Bi[k]; P.Ei[k] = (real)Ei[k]; }
    const double a2 = dh[1 * 4 + 1], a3 = dh[2 * 4 + 1], d4 = dh[3 * 4 + 0];
    P.d1 = (real)dh[0];
    P.D = (real)(dh[1 * 4 + 0] + dh[2 * 4 + 0]);
    P.a2 = (real)a2;
    P.k2 = (real)(a2 * a2 - a3 * a3 - d4 * d4);
    P.two_a2 = (real)(2 * a2);
    P.beta3 = (real)atan2(a3, d4);
    P.sign_a2 = a2 > 0 ? (real)1 : (real)-1;
    for (int j = 0; j < 6; j++) P.off[j] = (real)dh[j * 4 + 3];
    P.wrist_neg = dh[3 * 4 + 2] > 0;
    for (int k = 0; k < 8; k++) P.conf[k] = k < nconf ? conf[k] : 0;
    P.vec = ((uintptr_t)T & 15) == 0;
    P.nrows = N;
    const unsigned blocks = (unsigned)((N + 32 * B2K_IK6_WARPS - 1) / (32 * B2K_IK6_WARPS));
    switch (nconf) {
#define B2K_CASE(NC) \
    case NC: k_ikine_6s<real, NC><<<blocks, 32 * B2K_IK6_WARPS, 0, st>>>(P, (const real *)T, (real *)q, (int *)ok); break;
        B2K_CASE(1) B2K_CASE(2) B2K_CASE(3) B2K_CASE(4) B2K_CASE(5) B2K_CASE(6) B2K_CASE(7) B2K_CASE(8)
#undef B2K_CASE
    }
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

} // namespace

extern "C" int b2k_ikine_6s(int dtype, const double *dh, const double *base, const double *tool, const void *T, int64_t N, int nconf,
                            const int32_t *conf, void *q, int32_t *ok, void *stream)
{
    const char *fn = "b2k_ikine_6s";
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: bad N", fn); return B2K_ERR_INVALID; }
    if (nconf < 1 || nconf > 8) { b2k_set_error("%s: nconf must be 1..8, got %d", fn, nconf); return B2K_ERR_INVALID; }
    if (!dh || !conf) { b2k_set_error("%s: dh and conf must not be NULL", fn); return B2K_ERR_INVALID; }
    if (N > 0 && (!T || !q || !ok)) { b2k_set_error("%s: T, q and ok must not be NULL", fn); return B2K_ERR_INVALID; }
    for (int k = 0; k < nconf; k++)
        if (conf[k] < 0 || conf[k] > 7) { b2k_set_error("%s: configuration code %d of slot %d is not 0..7", fn, conf[k], k); return B2K_ERR_INVALID; }
    for (int e = 0; e < 24; e++)
        if (!isfinite(dh[e])) { b2k_set_error("%s: dh[%d][%d] is not finite", fn, e / 4, e % 4); return B2K_ERR_INVALID; }
    // the Puma link pattern, link by link; NaN-safe comparisons
    const double h = 1.5707963267948966, tol = 1e-9;
    const double *d = dh, *a = dh + 1, *al = dh + 2; // stride 4
    const struct { bool bad; const char *what; double got; } pattern[] = {
        {!(fabs(al[0] - h) <= tol), "alpha1 must be +pi/2", al[0]},
        {!(fabs(a[0]) <= tol), "a1 must be 0", a[0]},
        {!(fabs(al[4]) <= tol), "alpha2 must be 0", al[4]},
        {!(fabs(a[4]) > tol), "a2 must not be 0", a[4]},
        {!(fabs(al[8] + h) <= tol), "alpha3 must be -pi/2", al[8]},
        {!(fabs(fabs(al[12]) - h) <= tol), "alpha4 must be +pi/2 or -pi/2", al[12]},
        {!(fabs(a[12]) <= tol), "a4 must be 0", a[12]},
        {!(fabs(al[16] + al[12]) <= tol), "alpha5 must be -alpha4", al[16]},
        {!(fabs(a[16]) <= tol), "a5 must be 0", a[16]},
        {!(fabs(d[16]) <= tol), "d5 must be 0", d[16]},
    };
    for (const auto &p : pattern)
        if (p.bad) {
            b2k_set_error("%s: not a Puma-type arm: %s (got %.17g); the closed form needs alpha = (pi/2, 0, -pi/2, +-pi/2, "
                          "-+pi/2, any), a1 = a4 = a5 = 0, d5 = 0, a2 != 0", fn, p.what, p.got);
            return B2K_ERR_INVALID;
        }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(T);
    // fold the constants on the host in fp64: Bi = base^-1, Ei = tool^-1 Tt^-1 = (Tt tool)^-1
    double Bt[12], Tt[12], E[12], Bi[12], Ei[12], tl[12];
    b2k_ident34(Bt);
    if (base) b2k_mat_to34(base, Bt);
    const double a6 = a[20], d6 = d[20], ca = cos(al[20]), sa = sin(al[20]);
    const double Tt_[12] = {1, 0, 0, a6, 0, ca, -sa, 0, 0, sa, ca, d6};
    for (int k = 0; k < 12; k++) Tt[k] = Tt_[k];
    b2k_ident34(tl);
    if (tool) b2k_mat_to34(tool, tl);
    b2k_mul34(Tt, tl, E);
    ik6_inv_rigid(Bt, Bi);
    ik6_inv_rigid(E, Ei);
    cudaStream_t st = (cudaStream_t)stream;
    return dtype == B2K_F64 ? ik6_launch<double>(Bi, Ei, dh, T, N, nconf, conf, q, ok, st)
                            : ik6_launch<float>(Bi, Ei, dh, T, N, nconf, conf, q, ok, st);
}
