// b2k_ik6s.cu -- closed-form inverse kinematics over a batch of poses, every requested shoulder / elbow / wrist
// configuration from one read of each pose: Puma-type 6R arms with a spherical wrist (k_ikine_6s, the reference's
// DHRobot.ikine_6s / Puma560.ikine_a), UR-type 6R arms with three parallel axes (k_ikine_ur, DHRobot.ikine_ur) and
// Panda-type 7R arms at a given q7 (k_ikine_panda, DHRobot.ikine_panda).
//
// One lane per row, 64-thread blocks.  Each warp stages its 32 poses through shared memory with 16-byte loads (odd row
// pitch, so the lanes then read their own rows without bank conflicts), and the same stage then collects the (nconf, NJ)
// joint rows and the ok flags so that they leave coalesced (ik6_tile, NJ = 6 or 7).  The 6R arms work in the folded frame
// W = base^-1 T tool^-1 Tt^-1, Tt = transl(a6, 0, d6) Rx(alpha6), folded on the host into two constant 3x4 matrices.
//
// Puma: per row the wrist centre W, its distance r from the first axis and atan2(Py, Px) are formed once; per shoulder
// theta1, V, the elbow cosine and Rz(theta1)^T R(W); per configuration the rest.  With the pattern's twists
// R(A1 A2 A3) = Rz(theta1) Ry(-(theta2 + theta3)), so R(A1 A2 A3)^T R(W) is two plane rotations of R(W), not three link
// products.  DESIGN (f-6) states the algorithm and what the configuration letters mean.
//
// UR: W = A1 ... A5 Rz(theta6), so W's origin is O5.  Per row r and atan2(Py, Px); per shoulder theta1 and the first
// joint axis z1 in W's columns, (u, v, w) = (s5 c6, -s5 s6, c5); per configuration theta5 and theta6 from (u, v, w),
// then O4 and the axis x4, which reduce the parallel axes 2, 3 and 4 to a planar two-link problem.  DESIGN (f-15).
//
// Panda (modified DH): W = (base Rx(alpha1) Tx(a1))^-1 T (Tz(d7) tool)^-1 Rz(-theta7) (Rx(alpha7) Tx(a7))^-1 is frame 6,
// two host-folded constants around one per-row rotation by theta7 = q7 + offset7, read from the row's q7.  Per row
// v = O6 -> O2 in frame 6, h, psi and the elbow's acos; per elbow theta4, the frame-4 triangle (r, p) and the wrist's
// angle; per configuration theta6, theta5 and the ZYZ Euler angles of R3 = R(W) R(A6)^T R(A5)^T R(A4)^T, three column
// rotations of R(W).  DESIGN (f-17).
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

template <typename real>
struct IkurP {
    real Bi[12];           // base^-1, 3x4 row-major
    real Ei[12];           // tool^-1 Tt^-1, Tt = transl(a6, 0, d6) Rx(alpha6)
    real d1, D, d5;        // D = d2 + d3 + d4
    real a2, a3, k3, inv3; // k3 = a2^2 + a3^2, inv3 = 1 / (2 a2 a3)
    real sign_a23;         // sign(a2 a3)
    real off[6];
    int conf[8];
    int vec;               // T is 16-byte aligned
    long long nrows;
};

template <typename real>
struct IkpandaP {
    real Bi[12];         // (base Rx(alpha1) Tx(a1))^-1, 3x4 row-major
    real Ei[12];         // (Tz(d7) tool)^-1
    real Fi[12];         // (Rx(alpha7) Tx(a7))^-1
    real d1, K, hirho;   // K = a4^2 + d3^2 + a5^2 + d5^2, hirho = 1 / (2 rho)
    real phi, a4, d3, a5, d5;
    real off[7];
    const real *q7;      // (N,) device
    int conf[8];
    int vec;             // T is 16-byte aligned
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

// sin and cos of the angles these kernels form, all below 8 pi in magnitude (or NaN on a row that is out of reach):
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

// One warp's tile of 32 rows: stage the poses, hand each lane the top 3x4 of its pose, let solve(t, row, qs, oks) write
// the row's NC joint vectors of NJ joints to qs[NJ k + j] and its NC flags to oks[k] in the stage, then store both
// coalesced.  Idle lanes of a ragged tile solve the tile's first row into their own stage slots, which are never stored.
template <typename real, int NJ, int NC, typename Solve>
__device__ __forceinline__ void ik6_tile(int vec, long long nrows, const real *__restrict__ T, real *__restrict__ q,
                                         int *__restrict__ ok, const Solve &solve)
{
    constexpr int TS = 17;                   // odd pitch of a staged pose row
    constexpr int QW = NJ * NC, QS = QW | 1; // a row of q, and its odd pitch in the stage
    constexpr int OS = NC | 1;               // odd pitch of a row of ok flags
    constexpr int SS = TS > QS ? TS : QS;
    __shared__ real stage[B2K_IK6_WARPS][32 * SS];
    __shared__ int okst[B2K_IK6_WARPS][32 * OS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long row0 = ((long long)blockIdx.x * B2K_IK6_WARPS + warp) * 32;
    if (row0 >= nrows) return;
    const int rows = (int)(nrows - row0 < 32 ? nrows - row0 : 32);
    real *st = stage[warp];
    int *so = okst[warp];

    const real *src = T + row0 * 16;
    if (vec) {
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
    const int lr = lane < rows ? lane : 0;
    real t[12];
#pragma unroll
    for (int k = 0; k < 12; k++) t[k] = st[lr * TS + k];
    __syncwarp(); // the stage now collects the output
    solve(t, row0 + lr, st + lane * QS, so + lane * OS);
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

template <typename real, int NC>
__global__ void __launch_bounds__(32 * B2K_IK6_WARPS) k_ikine_6s(const __grid_constant__ Ik6sP<real> P, const real *__restrict__ T,
                                                                  real *__restrict__ q, int *__restrict__ ok)
{
    ik6_tile<real, 6, NC>(P.vec, P.nrows, T, q, ok, [&](const real *t, long long, real *qs, int *oks) {
        real M[12], W[12];
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
            for (int j = 0; j < 6; j++) qs[k * 6 + j] = good ? ik6_wrap<real>(th[j] - P.off[j]) : (real)NAN;
            oks[k] = good;
        }
    });
}

// |c3| up to 1 + B2K_IKUR_ELBOW_BAND eps of the compute type counts as reached and is clamped to 1: a straight elbow
// (UR10's qz and qr) has c3 = +-1 only up to the rounding of the fold and of X^2 + Y^2
#define B2K_IKUR_ELBOW_BAND 64

template <typename real, int NC>
__global__ void __launch_bounds__(32 * B2K_IK6_WARPS) k_ikine_ur(const __grid_constant__ IkurP<real> P, const real *__restrict__ T,
                                                                  real *__restrict__ q, int *__restrict__ ok)
{
    ik6_tile<real, 6, NC>(P.vec, P.nrows, T, q, ok, [&](const real *t, long long, real *qs, int *oks) {
        real M[12], W[12]; // W = A1 ... A5 Rz(theta6): columns x', y', z', origin O5
        ik6_mul34<real>(P.Bi, t, M);
        ik6_mul34<real>(M, P.Ei, W);
        const real pi = (real)3.14159265358979323846, eps = r_eps<real>();
        const Ik6SinCos sc;
        const real px = W[3], py = W[7], pz = W[11];
        const real r = hypot(px, py);
        const bool reach = fabs(P.D) <= r;
        const real phi = r_atan2<real>(py, px), s = asin(P.D / r);
        // per shoulder (index 0 = l, 1 = r): theta1, x1 = (c1, s1, 0), and z1 = (s1, -c1, 0) against W's columns
        real th1[2], c1[2], s1[2], uu[2], vv[2], ww[2];
#pragma unroll
        for (int sh = 0; sh < 2; sh++) {
            th1[sh] = phi + (sh ? s : pi - s);
            sc(th1[sh], s1[sh], c1[sh]);
            uu[sh] = W[0] * s1[sh] - W[4] * c1[sh];
            vv[sh] = W[1] * s1[sh] - W[5] * c1[sh];
            ww[sh] = W[2] * s1[sh] - W[6] * c1[sh];
        }

#pragma unroll 1
        for (int k = 0; k < NC; k++) {
            const int code = P.conf[k];
            const bool right = code & 1, down = code & 2, flip = code & 4;
            // ternaries, not a run-time index, keep the per-shoulder values in registers
            const real t1 = right ? th1[1] : th1[0], ca = right ? c1[1] : c1[0], sa = right ? s1[1] : s1[0];
            const real u = right ? uu[1] : uu[0], v = right ? vv[1] : vv[0], w = right ? ww[1] : ww[0];
            // wrist: (u, v, w) = (s5 c6, -s5 s6, c5), sigma = sign(s5) = +1 for "n", -1 for "f"
            const real sg = flip ? (real)-1 : (real)1, h = hypot(u, v);
            const bool sing = fabs(u) < 10 * eps && fabs(v) < 10 * eps; // theta6 = 0, as tr2eul's singular rule
            const real th5 = r_atan2<real>(sg * h, w), th6 = sing ? (real)0 : r_atan2<real>(-sg * v, sg * u);
            const real ih = sg / h;
            const real s5 = sg * h, c5 = w, c6 = sing ? (real)1 : u * ih, s6 = sing ? (real)0 : -v * ih;
            // the planar problem: O4 = O5 + d5 (s6 x' + c6 y'), X = O4 . x1, Y = O4z - d1; x4 = c5 (c6 x' - s6 y') - s5 z'
            const real o0 = px + P.d5 * (s6 * W[0] + c6 * W[1]);
            const real o1 = py + P.d5 * (s6 * W[4] + c6 * W[5]);
            const real o2 = pz + P.d5 * (s6 * W[8] + c6 * W[9]);
            const real X = o0 * ca + o1 * sa, Y = o2 - P.d1;
            const real x40 = c5 * (c6 * W[0] - s6 * W[1]) - s5 * W[2];
            const real x41 = c5 * (c6 * W[4] - s6 * W[5]) - s5 * W[6];
            const real x42 = c5 * (c6 * W[8] - s6 * W[9]) - s5 * W[10];
            const real th234 = r_atan2<real>(x42, x40 * ca + x41 * sa);
            // elbow: theta3 = -+sign(X) sign(a2 a3) acos(c3) for u / d, with sign(0) = +1
            const real c3r = (X * X + Y * Y - P.k3) * P.inv3;
            const bool good = reach && fabs(c3r) <= 1 + B2K_IKUR_ELBOW_BAND * eps; // false for NaN too
            const real c3 = fmin(fmax(c3r, (real)-1), (real)1);
            const real sgn3 = ((X >= 0) == down ? (real)1 : (real)-1) * P.sign_a23;
            const real th3 = sgn3 * acos(c3), s3 = sgn3 * sqrt((1 - c3) * (1 + c3));
            // theta2 = atan2(Y, X) - atan2(a3 s3, a2 + a3 c3), as one atan2 of the difference
            const real ex = fma(P.a3, c3, P.a2), ey = P.a3 * s3;
            const real th2 = r_atan2<real>(Y * ex - X * ey, X * ex + Y * ey);
            const real th[6] = {t1, th2, th3, th234 - th2 - th3, th5, th6};
#pragma unroll
            for (int j = 0; j < 6; j++) qs[k * 6 + j] = good ? ik6_wrap<real>(th[j] - P.off[j]) : (real)NAN;
            oks[k] = good;
        }
    });
}

// |C / rho| of the elbow up to 1 + B2K_IKPANDA_BAND eps of the compute type, and |p| of the wrist up to h +
// B2K_IKPANDA_BAND eps |v|, count as reached and are clamped: on-boundary rows (theta4 = phi or phi + pi, theta5 =
// +-pi/2) reach the boundary only up to the rounding of the fold, of |v|^2 and of the elbow triangle.  The wrist's band
// is a length, because p / h overshoots by eps |v| / h where O2 nears joint 6's axis (DESIGN f-17)
#define B2K_IKPANDA_BAND 64

// (m0 m1 m2) <- (m0 m1 m2) Rz(-theta) Rx(sg pi/2) on the columns of a 3x3, with c, s = cos, sin theta and sg = +-1
template <typename real>
__device__ __forceinline__ void ikp_cols(real (&m)[3][3], real c, real s, real sg)
{
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const real n0 = c * m[i][0] - s * m[i][1], n1 = s * m[i][0] + c * m[i][1], n2 = m[i][2];
        m[i][0] = n0;
        m[i][1] = sg * n2;
        m[i][2] = -sg * n1;
    }
}

template <typename real, int NC>
__global__ void __launch_bounds__(32 * B2K_IK6_WARPS) k_ikine_panda(const __grid_constant__ IkpandaP<real> P, const real *__restrict__ T,
                                                                     real *__restrict__ q, int *__restrict__ ok)
{
    ik6_tile<real, 7, NC>(P.vec, P.nrows, T, q, ok, [&](const real *t, long long row, real *qs, int *oks) {
        const real pi = (real)3.14159265358979323846, eps = r_eps<real>();
        const Ik6SinCos sc;
        const real q7 = __ldg(P.q7 + row);
        // W = Bi T Ei Rz(-theta7) Fi = A2 ... A6: frame 6, whose origin is the wrist point O6 = O5
        real M[12], E[12], G[12], W[12];
        ik6_mul34<real>(P.Bi, t, M);
        ik6_mul34<real>(M, P.Ei, E);
        real s7, c7;
        sc(q7 + P.off[6], s7, c7);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            G[j] = c7 * P.Fi[j] + s7 * P.Fi[4 + j];
            G[4 + j] = c7 * P.Fi[4 + j] - s7 * P.Fi[j];
            G[8 + j] = P.Fi[8 + j];
        }
        ik6_mul34<real>(E, G, W);
        // v = O6 -> O2 in frame 6, O2 = (0, 0, d1)
        const real e0 = -W[3], e1 = -W[7], e2 = P.d1 - W[11];
        const real vx = W[0] * e0 + W[4] * e1 + W[8] * e2;
        const real vy = W[1] * e0 + W[5] * e1 + W[9] * e2;
        const real vz = W[2] * e0 + W[6] * e1 + W[10] * e2;
        const real vv = vx * vx + vy * vy + vz * vz, h = hypot(vx, vy);
        // h at the rounding of |v|: O2 on joint 6's axis, theta6 free; psi = 0 and the wrist equation reads p = 0
        const real vn = sqrt(vv), tiny = 16 * eps * vn;
        const bool axis6 = h <= tiny;
        const real psi = axis6 ? (real)0 : r_atan2<real>(vy, vx);
        // elbow: theta4 = phi +- acos(C / rho)
        const real cr = (P.K - vv) * P.hirho;
        const bool reach = isfinite(q7) && fabs(cr) <= 1 + B2K_IKPANDA_BAND * eps; // false for NaN too
        const real ac = acos(fmin(fmax(cr, (real)-1), (real)1));
        // per elbow (index 0 = u, 1 = d): theta4, (r, p) = O6 -> O2 in frame 4's x and y, and theta6 + psi = asin(p / h)
        // as atan2(p, w) with w = c5 r = sqrt(h^2 - p^2) = sqrt(r^2 - v_z^2), from the difference of the smaller squares:
        // near O2 on joint 5's axis (r -> 0, theta5 free) h^2 - p^2 would leave w, and theta6, at the square root of the
        // rounding.  |r| at the rounding of |v| counts as on that axis.
        real th4[2], c4[2], s4[2], rr[2], as[2];
        bool wr_ok[2], axis5[2];
#pragma unroll
        for (int el = 0; el < 2; el++) {
            th4[el] = P.phi + (el ? -ac : ac);
            sc(th4[el], s4[el], c4[el]);
            rr[el] = -P.a4 * c4[el] - P.d3 * s4[el] - P.a5;
            const real p = P.a4 * s4[el] - P.d3 * c4[el] - P.d5;
            axis5[el] = fabs(rr[el]) <= tiny;
            wr_ok[el] = fabs(p) - h <= B2K_IKPANDA_BAND * eps * vn;
            const real w2 = fabs(rr[el]) < h ? (rr[el] - vz) * (rr[el] + vz) : (h - p) * (h + p);
            as[el] = axis6 ? (real)0 : r_atan2<real>(p, sqrt(fmax(w2, (real)0)));
        }

#pragma unroll 1
        for (int k = 0; k < NC; k++) {
            const int code = P.conf[k];
            const bool right = code & 1, down = code & 2, flip = code & 4;
            // ternaries, not a run-time index, keep the per-elbow values in registers
            const real t4 = down ? th4[1] : th4[0], ca4 = down ? c4[1] : c4[0], sa4 = down ? s4[1] : s4[0];
            const real r = down ? rr[1] : rr[0], a6 = down ? as[1] : as[0];
            // wrist: v_x s6 + v_y c6 = p, then theta5 from the two remaining components, 0 where it is free
            const real th6 = (flip ? pi - a6 : a6) - psi;
            real s6, c6;
            sc(th6, s6, c6);
            const real sg = r >= 0 ? (real)1 : (real)-1, vu = vx * c6 - vy * s6;
            const real th5 = (down ? axis5[1] : axis5[0]) ? (real)0 : r_atan2<real>(sg * vz, sg * vu);
            real s5, c5;
            sc(th5, s5, c5);
            // shoulder: R3 = R(W) (Rx(pi/2) Rz(theta6))^T (Rx(-pi/2) Rz(theta5))^T (Rx(pi/2) Rz(theta4))^T, ZYZ Euler
            real R[3][3];
#pragma unroll
            for (int i = 0; i < 3; i++)
#pragma unroll
                for (int j = 0; j < 3; j++) R[i][j] = W[i * 4 + j];
            ikp_cols<real>(R, c6, s6, (real)-1);
            ikp_cols<real>(R, c5, s5, (real)1);
            ikp_cols<real>(R, ca4, sa4, (real)-1);
            real g[3];
            if (right) rot_to_eul<real, false, Ik6SinCos>(R, g);
            else rot_to_eul<real, true, Ik6SinCos>(R, g);
            const real th[6] = {g[0], g[1], g[2], t4, th5, th6};
            const bool good = reach && (down ? wr_ok[1] : wr_ok[0]);
#pragma unroll
            for (int j = 0; j < 6; j++) qs[k * 7 + j] = good ? ik6_wrap<real>(th[j] - P.off[j]) : (real)NAN;
            qs[k * 7 + 6] = good ? q7 : (real)NAN;
            oks[k] = good;
        }
    });
}

// inverse of a rigid 3x4 transform: [R^T | -R^T t]
void ik6_inv_rigid(const double *A, double *X)
{
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) X[i * 4 + j] = A[j * 4 + i];
        X[i * 4 + 3] = -(A[0 * 4 + i] * A[3] + A[1 * 4 + i] * A[7] + A[2 * 4 + i] * A[11]);
    }
}

// The checks every entry point makes before its link pattern, in this order, for a table of nj rows.  The per-row q7 of
// the 7R arms (nj = 7) must be non-NULL when N > 0 and aligned to its element size.  B2K_OK or B2K_ERR_INVALID.
int ik6_check(const char *fn, int dtype, int nj, const double *dh, const void *T, const void *q7, int64_t N, int nconf,
              const int32_t *conf, const void *q, const int32_t *ok)
{
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: bad N", fn); return B2K_ERR_INVALID; }
    if (nconf < 1 || nconf > 8) { b2k_set_error("%s: nconf must be 1..8, got %d", fn, nconf); return B2K_ERR_INVALID; }
    if (!dh || !conf) { b2k_set_error("%s: dh and conf must not be NULL", fn); return B2K_ERR_INVALID; }
    if (N > 0 && (!T || !q || !ok)) { b2k_set_error("%s: T, q and ok must not be NULL", fn); return B2K_ERR_INVALID; }
    if (nj == 7 && N > 0 && !q7) { b2k_set_error("%s: q7 must not be NULL", fn); return B2K_ERR_INVALID; }
    if (nj == 7 && ((uintptr_t)q7 % (dtype == B2K_F64 ? 8 : 4))) { b2k_set_error("%s: q7 must be aligned to its element size", fn); return B2K_ERR_INVALID; }
    for (int k = 0; k < nconf; k++)
        if (conf[k] < 0 || conf[k] > 7) { b2k_set_error("%s: configuration code %d of slot %d is not 0..7", fn, conf[k], k); return B2K_ERR_INVALID; }
    for (int e = 0; e < nj * 4; e++)
        if (!isfinite(dh[e])) { b2k_set_error("%s: dh[%d][%d] is not finite", fn, e / 4, e % 4); return B2K_ERR_INVALID; }
    return B2K_OK;
}

struct Ik6Rule {
    bool bad;
    const char *what;
    double got;
};

// the first broken rule of a link pattern as "<fn>: not a <arm>-type arm: <what> (got <value>); <needs>"
template <size_t R>
int ik6_pattern(const char *fn, const Ik6Rule (&rules)[R], const char *arm, const char *needs)
{
    for (const auto &p : rules)
        if (p.bad) {
            b2k_set_error("%s: not a %s-type arm: %s (got %.17g); the closed form needs %s", fn, arm, p.what, p.got, needs);
            return B2K_ERR_INVALID;
        }
    return B2K_OK;
}

// fold the constants on the host in fp64: Bi = (base head)^-1, Ei = (Tt tool)^-1; base, head and tool NULL = identity.
// The 6R arms have no head and Tt = transl(a6, 0, d6) Rx(alpha6) (ik6_tail).
void ik6_fold(const double *base, const double *head, const double *Tt, const double *tool, double *Bi, double *Ei)
{
    double Bt[12], E[12], tl[12];
    b2k_ident34(Bt);
    if (base) b2k_mat_to34(base, Bt);
    if (head) {
        double X[12];
        b2k_mul34(Bt, head, X);
        for (int k = 0; k < 12; k++) Bt[k] = X[k];
    }
    b2k_ident34(tl);
    if (tool) b2k_mat_to34(tool, tl);
    b2k_mul34(Tt, tl, E);
    ik6_inv_rigid(Bt, Bi);
    ik6_inv_rigid(E, Ei);
}

// Tt = transl(a6, 0, d6) Rx(alpha6), the constant part of a standard-DH 6R arm's last link
void ik6_tail(const double *dh, double *Tt)
{
    const double a6 = dh[20 + 1], d6 = dh[20], ca = cos(dh[20 + 2]), sa = sin(dh[20 + 2]);
    const double X[12] = {1, 0, 0, a6, 0, ca, -sa, 0, 0, sa, ca, d6};
    for (int k = 0; k < 12; k++) Tt[k] = X[k];
}

// the fields every parameter block has, then one launch of kern[nconf - 1], the instantiation for nconf configurations
template <typename real, typename Prm>
int ik6_launch(void (*const kern[8])(Prm, const real *, real *, int *), Prm &P, const double *Bi, const double *Ei,
               const double *dh, const void *T, long long N, int nconf, const int32_t *conf, void *q, int32_t *ok,
               cudaStream_t st)
{
    constexpr int NJ = sizeof(P.off) / sizeof(P.off[0]);
    for (int k = 0; k < 12; k++) { P.Bi[k] = (real)Bi[k]; P.Ei[k] = (real)Ei[k]; }
    for (int j = 0; j < NJ; j++) P.off[j] = (real)dh[j * 4 + 3];
    for (int k = 0; k < 8; k++) P.conf[k] = k < nconf ? conf[k] : 0;
    P.vec = ((uintptr_t)T & 15) == 0;
    P.nrows = N;
    const unsigned blocks = (unsigned)((N + 32 * B2K_IK6_WARPS - 1) / (32 * B2K_IK6_WARPS));
    kern[nconf - 1]<<<blocks, 32 * B2K_IK6_WARPS, 0, st>>>(P, (const real *)T, (real *)q, (int *)ok);
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

template <typename real>
int ik6s_launch(const double *Bi, const double *Ei, const double *dh, const void *T, long long N, int nconf, const int32_t *conf,
                void *q, int32_t *ok, cudaStream_t st)
{
    static void (*const kern[8])(Ik6sP<real>, const real *, real *, int *) = {
        k_ikine_6s<real, 1>, k_ikine_6s<real, 2>, k_ikine_6s<real, 3>, k_ikine_6s<real, 4>,
        k_ikine_6s<real, 5>, k_ikine_6s<real, 6>, k_ikine_6s<real, 7>, k_ikine_6s<real, 8>};
    Ik6sP<real> P;
    const double a2 = dh[1 * 4 + 1], a3 = dh[2 * 4 + 1], d4 = dh[3 * 4 + 0];
    P.d1 = (real)dh[0];
    P.D = (real)(dh[1 * 4 + 0] + dh[2 * 4 + 0]);
    P.a2 = (real)a2;
    P.k2 = (real)(a2 * a2 - a3 * a3 - d4 * d4);
    P.two_a2 = (real)(2 * a2);
    P.beta3 = (real)atan2(a3, d4);
    P.sign_a2 = a2 > 0 ? (real)1 : (real)-1;
    P.wrist_neg = dh[3 * 4 + 2] > 0;
    return ik6_launch<real>(kern, P, Bi, Ei, dh, T, N, nconf, conf, q, ok, st);
}

template <typename real>
int ikur_launch(const double *Bi, const double *Ei, const double *dh, const void *T, long long N, int nconf, const int32_t *conf,
                void *q, int32_t *ok, cudaStream_t st)
{
    static void (*const kern[8])(IkurP<real>, const real *, real *, int *) = {
        k_ikine_ur<real, 1>, k_ikine_ur<real, 2>, k_ikine_ur<real, 3>, k_ikine_ur<real, 4>,
        k_ikine_ur<real, 5>, k_ikine_ur<real, 6>, k_ikine_ur<real, 7>, k_ikine_ur<real, 8>};
    IkurP<real> P;
    const double a2 = dh[1 * 4 + 1], a3 = dh[2 * 4 + 1];
    P.d1 = (real)dh[0];
    P.D = (real)(dh[1 * 4 + 0] + dh[2 * 4 + 0] + dh[3 * 4 + 0]);
    P.d5 = (real)dh[4 * 4 + 0];
    P.a2 = (real)a2;
    P.a3 = (real)a3;
    P.k3 = (real)(a2 * a2 + a3 * a3);
    P.inv3 = (real)(1 / (2 * a2 * a3));
    P.sign_a23 = a2 * a3 > 0 ? (real)1 : (real)-1;
    return ik6_launch<real>(kern, P, Bi, Ei, dh, T, N, nconf, conf, q, ok, st);
}

template <typename real>
int ikpanda_launch(const double *Bi, const double *Ei, const double *Fi, const double *dh, const void *T, const void *q7, long long N,
                   int nconf, const int32_t *conf, void *q, int32_t *ok, cudaStream_t st)
{
    static void (*const kern[8])(IkpandaP<real>, const real *, real *, int *) = {
        k_ikine_panda<real, 1>, k_ikine_panda<real, 2>, k_ikine_panda<real, 3>, k_ikine_panda<real, 4>,
        k_ikine_panda<real, 5>, k_ikine_panda<real, 6>, k_ikine_panda<real, 7>, k_ikine_panda<real, 8>};
    IkpandaP<real> P;
    const double d3 = dh[2 * 4 + 0], a4 = dh[3 * 4 + 1], a5 = dh[4 * 4 + 1], d5 = dh[4 * 4 + 0];
    const double A = -a4 * a5 - d3 * d5, B = a4 * d5 - d3 * a5;
    for (int k = 0; k < 12; k++) P.Fi[k] = (real)Fi[k];
    P.d1 = (real)dh[0];
    P.K = (real)(a4 * a4 + d3 * d3 + a5 * a5 + d5 * d5);
    P.hirho = (real)(0.5 / hypot(A, B));
    P.phi = (real)atan2(B, A);
    P.a4 = (real)a4;
    P.d3 = (real)d3;
    P.a5 = (real)a5;
    P.d5 = (real)d5;
    P.q7 = (const real *)q7;
    return ik6_launch<real>(kern, P, Bi, Ei, dh, T, N, nconf, conf, q, ok, st);
}

const double kHalfPi = 1.5707963267948966, kPatternTol = 1e-9;

} // namespace

extern "C" int b2k_ikine_6s(int dtype, const double *dh, const double *base, const double *tool, const void *T, int64_t N, int nconf,
                            const int32_t *conf, void *q, int32_t *ok, void *stream)
{
    const char *fn = "b2k_ikine_6s";
    if (int rc = ik6_check(fn, dtype, 6, dh, T, nullptr, N, nconf, conf, q, ok)) return rc;
    // the Puma link pattern, link by link; NaN-safe comparisons
    const double h = kHalfPi, tol = kPatternTol;
    const double *d = dh, *a = dh + 1, *al = dh + 2; // stride 4
    const Ik6Rule pattern[] = {
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
    if (int rc = ik6_pattern(fn, pattern, "Puma", "alpha = (pi/2, 0, -pi/2, +-pi/2, -+pi/2, any), a1 = a4 = a5 = 0, d5 = 0, a2 != 0"))
        return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(T);
    double Tt[12], Bi[12], Ei[12];
    ik6_tail(dh, Tt);
    ik6_fold(base, nullptr, Tt, tool, Bi, Ei);
    cudaStream_t st = (cudaStream_t)stream;
    return dtype == B2K_F64 ? ik6s_launch<double>(Bi, Ei, dh, T, N, nconf, conf, q, ok, st)
                            : ik6s_launch<float>(Bi, Ei, dh, T, N, nconf, conf, q, ok, st);
}

extern "C" int b2k_ikine_ur(int dtype, const double *dh, const double *base, const double *tool, const void *T, int64_t N, int nconf,
                            const int32_t *conf, void *q, int32_t *ok, void *stream)
{
    const char *fn = "b2k_ikine_ur";
    if (int rc = ik6_check(fn, dtype, 6, dh, T, nullptr, N, nconf, conf, q, ok)) return rc;
    // the UR link pattern, link by link; NaN-safe comparisons
    const double h = kHalfPi, tol = kPatternTol;
    const double *a = dh + 1, *al = dh + 2; // stride 4
    const Ik6Rule pattern[] = {
        {!(fabs(al[0] - h) <= tol), "alpha1 must be +pi/2", al[0]},
        {!(fabs(a[0]) <= tol), "a1 must be 0", a[0]},
        {!(fabs(al[4]) <= tol), "alpha2 must be 0", al[4]},
        {!(fabs(a[4]) > tol), "a2 must not be 0", a[4]},
        {!(fabs(al[8]) <= tol), "alpha3 must be 0", al[8]},
        {!(fabs(a[8]) > tol), "a3 must not be 0", a[8]},
        {!(fabs(al[12] - h) <= tol), "alpha4 must be +pi/2", al[12]},
        {!(fabs(a[12]) <= tol), "a4 must be 0", a[12]},
        {!(fabs(al[16] + h) <= tol), "alpha5 must be -pi/2", al[16]},
        {!(fabs(a[16]) <= tol), "a5 must be 0", a[16]},
    };
    if (int rc = ik6_pattern(fn, pattern, "UR", "alpha = (pi/2, 0, 0, pi/2, -pi/2, any), a1 = a4 = a5 = 0, a2 != 0, a3 != 0"))
        return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(T);
    double Tt[12], Bi[12], Ei[12];
    ik6_tail(dh, Tt);
    ik6_fold(base, nullptr, Tt, tool, Bi, Ei);
    cudaStream_t st = (cudaStream_t)stream;
    return dtype == B2K_F64 ? ikur_launch<double>(Bi, Ei, dh, T, N, nconf, conf, q, ok, st)
                            : ikur_launch<float>(Bi, Ei, dh, T, N, nconf, conf, q, ok, st);
}

extern "C" int b2k_ikine_panda(int dtype, const double *dh, const double *base, const double *tool, const void *T, const void *q7,
                               int64_t N, int nconf, const int32_t *conf, void *q, int32_t *ok, void *stream)
{
    const char *fn = "b2k_ikine_panda";
    if (int rc = ik6_check(fn, dtype, 7, dh, T, q7, N, nconf, conf, q, ok)) return rc;
    // the Panda link pattern in modified DH, link by link; NaN-safe comparisons
    const double h = kHalfPi, tol = kPatternTol;
    const double *d = dh, *a = dh + 1, *al = dh + 2; // stride 4
    const double l34 = hypot(a[12], d[8]), l55 = hypot(a[16], d[16]);
    const Ik6Rule pattern[] = {
        {!(fabs(al[4] + h) <= tol), "alpha2 must be -pi/2", al[4]},
        {!(fabs(a[4]) <= tol), "a2 must be 0", a[4]},
        {!(fabs(d[4]) <= tol), "d2 must be 0", d[4]},
        {!(fabs(al[8] - h) <= tol), "alpha3 must be +pi/2", al[8]},
        {!(fabs(a[8]) <= tol), "a3 must be 0", a[8]},
        {!(fabs(al[12] - h) <= tol), "alpha4 must be +pi/2", al[12]},
        {!(fabs(d[12]) <= tol), "d4 must be 0", d[12]},
        {!(l34 > tol), "hypot(a4, d3) must not be 0", l34},
        {!(fabs(al[16] + h) <= tol), "alpha5 must be -pi/2", al[16]},
        {!(l55 > tol), "hypot(a5, d5) must not be 0", l55},
        {!(fabs(al[20] - h) <= tol), "alpha6 must be +pi/2", al[20]},
        {!(fabs(a[20]) <= tol), "a6 must be 0", a[20]},
        {!(fabs(d[20]) <= tol), "d6 must be 0", d[20]},
    };
    if (int rc = ik6_pattern(fn, pattern, "Panda",
                             "modified DH with alpha2 .. alpha6 = (-pi/2, pi/2, pi/2, -pi/2, pi/2), a2 = a3 = a6 = 0, d2 = d4 = d6 = 0, "
                             "hypot(a4, d3) != 0, hypot(a5, d5) != 0"))
        return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(T);
    // head = Rx(alpha1) Tx(a1), Tt = Tz(d7), F = Rx(alpha7) Tx(a7): W = (base head)^-1 T (Tt tool)^-1 Rz(-theta7) F^-1
    const double c1 = cos(al[0]), s1 = sin(al[0]), c7 = cos(al[24]), s7 = sin(al[24]);
    const double head[12] = {1, 0, 0, a[0], 0, c1, -s1, 0, 0, s1, c1, 0};
    const double Tt[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, d[24]};
    const double F[12] = {1, 0, 0, a[24], 0, c7, -s7, 0, 0, s7, c7, 0};
    double Bi[12], Ei[12], Fi[12];
    ik6_fold(base, head, Tt, tool, Bi, Ei);
    ik6_inv_rigid(F, Fi);
    cudaStream_t st = (cudaStream_t)stream;
    return dtype == B2K_F64 ? ikpanda_launch<double>(Bi, Ei, Fi, dh, T, q7, N, nconf, conf, q, ok, st)
                            : ikpanda_launch<float>(Bi, Ei, Fi, dh, T, q7, N, nconf, conf, q, ok, st);
}
