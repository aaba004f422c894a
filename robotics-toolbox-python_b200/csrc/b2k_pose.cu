// b2k_pose.cu -- batch producers / consumers either side of the kinematics path: pose errors, the analytical Jacobian
// and trajectories (SURVEY 8f-2, 8f-3), one lane per row or one thread per (row, axis) element:
//   b2k_angle_axis         fknm.Angle_Axis (fknm.cpp:112-162 -> _angle_axis ik.cpp:241-286), batched
//   b2k_p_servo            tools/p_servo.py:46-106 with method="angle-axis": v = gain .* angle_axis(Te, Tep)
//   b2k_p_servo_rpy        tools/p_servo.py:46-106 with its default method="rpy": error in the end-effector frame,
//                          e = [t(Te^-1 Tep); tr2rpy(Te^-1 Tep, order="zyx")]
//   b2k_jacob0_analytical  ETS.jacob0_analytical (ETS.py:1570-1626): blkdiag(I, A^-1(Gamma(R))) J0 for the four
//                          rate representations rpy/xyz, rpy/zyx, eul (ZYZ), exp
//   b2k_jtraj              joint-space quintic blend (tools/trajectory.py:686-780)
//   b2k_mtraj              scalar quintic / trapezoidal profiles and their multi-axis form (tools/trajectory.py:271-684)
//   b2k_ctraj              Cartesian trajectory T0 -> T1 (tools/trajectory.py:782-841 -> SE3.interp: translation
//                          lerp + unit-quaternion slerp), the (N,4,4) batch is born in HBM where ik_LM consumes it
//   b2k_mstraj             the sample table of tools/trajectory.py:852-1152 (multi-segment multi-axis trajectory):
//                          quintic blends and linear segments planned on the host, evaluated per (row, axis) here
// The angle conventions (tr2rpy, tr2eul, rotvelxform, quaternion slerp) belong to spatialmath-python, which is not
// part of the reference tree: they are restated from its documented definitions -- R = Rz(yaw) Ry(pitch) Rx(roll) for
// "zyx", R = Rx(yaw) Ry(pitch) Rz(roll) for "xyz", R = Rz(phi) Ry(theta) Rz(psi) for "eul", v = theta k for "exp" --
// and pinned by properties (tests: the analytical Jacobian equals the finite-difference derivative of Gamma(R(q));
// interpolation end points and constant angular rate), not by the package itself.
#include <math.h>

#include <algorithm>
#include <initializer_list>
#include <type_traits>
#include <vector>

#include "b2k_common.cuh"
#include "b2k_ik.cuh" // ik_angle_axis

namespace {

// tr2rpy(order="zyx"): R = Rz(yaw) Ry(pitch) Rx(roll) -> (roll, pitch, yaw); at |R20| = 1 roll := 0
template <typename real>
__device__ __forceinline__ void rot_to_rpy_zyx(const real R[3][3], real g[3])
{
    if (fabs(fabs(R[2][0]) - 1) < 10 * r_eps<real>()) {
        g[0] = 0;
        g[2] = R[2][0] < 0 ? -r_atan2<real>(R[0][1], R[0][2]) : r_atan2<real>(-R[0][1], -R[0][2]);
        g[1] = -asin(fmin(fmax(R[2][0], (real)-1), (real)1));
    } else {
        g[0] = r_atan2<real>(R[2][1], R[2][2]);
        g[2] = r_atan2<real>(R[1][0], R[0][0]);
        g[1] = r_atan2<real>(-R[2][0], sqrt(R[0][0] * R[0][0] + R[1][0] * R[1][0]));
    }
}
// tr2rpy(order="xyz"): R = Rx(yaw) Ry(pitch) Rz(roll) -> (roll, pitch, yaw)
template <typename real>
__device__ __forceinline__ void rot_to_rpy_xyz(const real R[3][3], real g[3])
{
    if (fabs(fabs(R[0][2]) - 1) < 10 * r_eps<real>()) {
        g[0] = 0;
        g[2] = R[0][2] > 0 ? r_atan2<real>(R[2][1], R[1][1]) : -r_atan2<real>(R[1][0], R[2][0]);
        g[1] = asin(fmin(fmax(R[0][2], (real)-1), (real)1));
    } else {
        g[0] = -r_atan2<real>(R[0][1], R[0][0]);
        g[2] = -r_atan2<real>(R[1][2], R[2][2]);
        g[1] = r_atan2<real>(R[0][2], sqrt(R[0][0] * R[0][0] + R[0][1] * R[0][1]));
    }
}
// trlog: exponential coordinates v = theta * axis
template <typename real>
__device__ __forceinline__ void rot_to_exp(const real R[3][3], real g[3])
{
    const real lx = R[2][1] - R[1][2], ly = R[0][2] - R[2][0], lz = R[1][0] - R[0][1];
    const real ln = sqrt(lx * lx + ly * ly + lz * lz), tr = R[0][0] + R[1][1] + R[2][2];
    if (ln < (real)1e-9 * (sizeof(real) == 8 ? 1 : 1000)) {
        if (tr > 0) { g[0] = g[1] = g[2] = 0; }
        else { // theta = pi: axis from the diagonal
            const real pi = (real)3.14159265358979323846;
            real ax = sqrt(fmax((R[0][0] + 1) / 2, (real)0)), ay = sqrt(fmax((R[1][1] + 1) / 2, (real)0)), az = sqrt(fmax((R[2][2] + 1) / 2, (real)0));
            if (ax >= ay && ax >= az) { ay = copysign(ay, R[0][1]); az = copysign(az, R[0][2]); }
            else if (ay >= az) { ax = copysign(ax, R[0][1]); az = copysign(az, R[1][2]); }
            else { ax = copysign(ax, R[0][2]); ay = copysign(ay, R[1][2]); }
            g[0] = pi * ax; g[1] = pi * ay; g[2] = pi * az;
        }
        return;
    }
    const real ang = r_atan2<real>(ln, tr - 1);
    g[0] = ang * lx / ln; g[1] = ang * ly / ln; g[2] = ang * lz / ln;
}

enum { REP_RPY_XYZ = 0, REP_RPY_ZYX = 1, REP_EUL = 2, REP_EXP = 3 };

// A^-1(Gamma): angular velocity -> representation rates (rotvelxform(..., inverse=True))
template <typename real>
__device__ __forceinline__ void rotvel_inverse(int rep, const real g[3], real A[3][3])
{
    if (rep == REP_RPY_ZYX) { // omega = yaw' z + pitch' Rz y + roll' Rz Ry x
        const real sb = sin(g[1]), cb = cos(g[1]), sg = sin(g[2]), cg = cos(g[2]), tb = sb / cb;
        A[0][0] = cg / cb; A[0][1] = sg / cb; A[0][2] = 0;
        A[1][0] = -sg;     A[1][1] = cg;      A[1][2] = 0;
        A[2][0] = cg * tb; A[2][1] = sg * tb; A[2][2] = 1;
    } else if (rep == REP_RPY_XYZ) { // omega = yaw' x + pitch' Rx y + roll' Rx Ry z
        const real sb = sin(g[1]), cb = cos(g[1]), sg = sin(g[2]), cg = cos(g[2]), tb = sb / cb;
        A[0][0] = 0; A[0][1] = -sg / cb; A[0][2] = cg / cb;
        A[1][0] = 0; A[1][1] = cg;       A[1][2] = sg;
        A[2][0] = 1; A[2][1] = sg * tb;  A[2][2] = -cg * tb;
    } else if (rep == REP_EUL) { // omega = phi' z + theta' Rz y + psi' Rz Ry z
        const real sp = sin(g[0]), cp = cos(g[0]), st = sin(g[1]), ct = cos(g[1]);
        A[0][0] = -cp * ct / st; A[0][1] = -sp * ct / st; A[0][2] = 1;
        A[1][0] = -sp;           A[1][1] = cp;            A[1][2] = 0;
        A[2][0] = cp / st;       A[2][1] = sp / st;       A[2][2] = 0;
    } else { // exponential coordinates: A^-1 = I - [v]x / 2 + k2 [v]x^2, k2 = (1 - x cot x) / theta^2, x = theta / 2
        // The equal form (1 - x sin(theta) / (1 - cos(theta))) / theta^2 loses the digits of 1 - cos(theta) to
        // cancellation at small theta (fp32: cos rounds to 1 below theta ~ 3.5e-4 and k2 is -inf).  Below theta0 (0.1
        // fp64, 0.5 fp32) the series, whose first omitted term theta^8 / 47900160 is below the dtype's rounding there;
        // above it 1 - x cot x >= theta0^2 / 12 loses a few bits, which the factor theta^2 of [v]x^2 gives back.
        const real th2 = g[0] * g[0] + g[1] * g[1] + g[2] * g[2], th = sqrt(th2);
        real k2;
        if (th < (sizeof(real) == 8 ? (real)0.1 : (real)0.5))
            k2 = (real)1 / 12 + th2 * ((real)1 / 720 + th2 * ((real)1 / 30240 + th2 * ((real)1 / 1209600)));
        else {
            const real x = th / 2;
            k2 = (1 - x * cos(x) / sin(x)) / th2;
        }
        const real S[3][3] = {{0, -g[2], g[1]}, {g[2], 0, -g[0]}, {-g[1], g[0], 0}};
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
                real s2 = 0;
                for (int k = 0; k < 3; k++) s2 += S[i][k] * S[k][j];
                A[i][j] = (i == j ? (real)1 : (real)0) - S[i][j] / 2 + k2 * s2;
            }
    }
}

// One lane per row; the warp stages its 32 Jacobian rows through shared memory (coalesced both ways) and converts them
// in place: the translational rows pass through, the rotational ones are multiplied by A^-1(Gamma(R)).
// Shared memory is sized for the robot at hand (2 warps x 32 rows x 6n reals: 21.5 KB at n = 7 fp64, 10 resident blocks
// per SM; a tile sized for B2K_MAX_JOINTS held the kernel to 7).
template <typename real, bool VEC>
__global__ void __launch_bounds__(64) k_janalytical(const real *__restrict__ T, const real *__restrict__ J, long long nrows, int n,
                                                    int rep, real *__restrict__ Ja)
{
    extern __shared__ __align__(16) unsigned char jan_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long row0 = ((long long)blockIdx.x * 2 + warp) * 32;
    if (row0 >= nrows) return;
    const int rows = (int)(nrows - row0 < 32 ? nrows - row0 : 32), w = 6 * n;
    real *tl = reinterpret_cast<real *>(jan_smem) + warp * 32 * w;
    for (int e = lane; e < rows * w; e += 32) tl[e] = J[row0 * w + e];
    __syncwarp();
    if (lane < rows) {
        real t[12];
        if (VEC) {
            load12<real>(T + (row0 + lane) * 16, t);
        } else {
#pragma unroll
            for (int k = 0; k < 12; k++) t[k] = T[(row0 + lane) * 16 + k];
        }
        real R[3][3], g[3], A[3][3];
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) R[i][j] = t[i * 4 + j];
        if (rep == REP_RPY_ZYX) rot_to_rpy_zyx<real>(R, g);
        else if (rep == REP_RPY_XYZ) rot_to_rpy_xyz<real>(R, g);
        else if (rep == REP_EUL) rot_to_eul<real>(R, g);
        else rot_to_exp<real>(R, g);
        rotvel_inverse<real>(rep, g, A);
        real *j = tl + lane * w;
        for (int c = 0; c < n; c++) {
            const real w0 = j[3 * n + c], w1 = j[4 * n + c], w2 = j[5 * n + c];
#pragma unroll
            for (int i = 0; i < 3; i++) j[(3 + i) * n + c] = A[i][0] * w0 + A[i][1] * w1 + A[i][2] * w2;
        }
    }
    __syncwarp();
    for (int e = lane; e < rows * w; e += 32) Ja[row0 * w + e] = tl[e];
}

// The pose error of Te against Tep, lane per row; tep_stride = 0 broadcasts one target to every row.
//   ERR_ANGLE_AXIS  e = angle_axis(Te, Tep)
//   ERR_RPY_ZYX     e = [Re^T (tp - te); rpy_zyx(Re^T Rep)]
// Then v = gain .* e and arrived = sum |e| < threshold (arrived may be NULL).
enum { ERR_ANGLE_AXIS = 0, ERR_RPY_ZYX = 1 };

template <typename real, bool VEC, int ERR>
__global__ void __launch_bounds__(256) k_pose_servo(const real *__restrict__ Te, const real *__restrict__ Tep, long long tep_stride,
                                                    long long nrows, real g0, real g1, real g2, real g3, real g4, real g5,
                                                    real threshold, real *__restrict__ out, int *__restrict__ arrived)
{
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    // the three used rows of both poses as 16-byte vector loads where both arrays are 16-byte aligned (the launcher
    // looks; any torch allocation is): a third of the load instructions of the scalar form
    real a[12], b[12], e[6];
    if (VEC) {
        load12<real>(Te + row * 16, a);
        load12<real>(Tep + row * tep_stride, b);
    } else {
#pragma unroll
        for (int k = 0; k < 12; k++) { a[k] = Te[row * 16 + k]; b[k] = Tep[row * tep_stride + k]; }
    }
    if constexpr (ERR == ERR_ANGLE_AXIS) {
        Pose<real> T;
        pose_from_const<real>(T, a);
        ik_angle_axis<real>(T, b, e);
    } else {
        real R[3][3];
        const real d[3] = {b[3] - a[3], b[7] - a[7], b[11] - a[11]};
#pragma unroll
        for (int i = 0; i < 3; i++) {
            e[i] = a[0 * 4 + i] * d[0] + a[1 * 4 + i] * d[1] + a[2 * 4 + i] * d[2];
#pragma unroll
            for (int j = 0; j < 3; j++) R[i][j] = a[0 * 4 + i] * b[0 * 4 + j] + a[1 * 4 + i] * b[1 * 4 + j] + a[2 * 4 + i] * b[2 * 4 + j];
        }
        rot_to_rpy_zyx<real>(R, e + 3);
    }
    const real g[6] = {g0, g1, g2, g3, g4, g5};
    real sum = 0;
#pragma unroll
    for (int k = 0; k < 6; k++) {
        sum += fabs(e[k]);
        out[row * 6 + k] = g[k] * e[k];
    }
    if (arrived) arrived[row] = sum < threshold ? 1 : 0;
}

struct CtrajP {
    double q0[4], q1[4]; // unit quaternions (s, x, y, z); q0 already negated for the shortest arc
    double theta, sin_theta;
    double p0[3], p1[3];
    int lerp_only; // the two orientations coincide
};

template <typename real, bool VEC>
__global__ void __launch_bounds__(256) k_ctraj(const __grid_constant__ CtrajP P, const real *__restrict__ s, long long nrows,
                                               real *__restrict__ T)
{
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    real u = s[row];
    u = fmin(fmax(u, (real)0), (real)1); // SE3.interp clips s to [0, 1]
    real q[4];
    if (u == 0 || P.lerp_only) { for (int k = 0; k < 4; k++) q[k] = (real)P.q0[k]; }
    else if (u == 1) { for (int k = 0; k < 4; k++) q[k] = (real)P.q1[k]; }
    else {
        const real th = (real)P.theta;
        const real s0 = sin((1 - u) * th) / (real)P.sin_theta, s1 = sin(u * th) / (real)P.sin_theta;
        for (int k = 0; k < 4; k++) q[k] = (real)P.q0[k] * s0 + (real)P.q1[k] * s1;
    }
    const real w = q[0], x = q[1], y = q[2], z = q[3];
    real o[16];
    o[0] = 1 - 2 * (y * y + z * z); o[1] = 2 * (x * y - w * z);     o[2] = 2 * (x * z + w * y);
    o[4] = 2 * (x * y + w * z);     o[5] = 1 - 2 * (x * x + z * z); o[6] = 2 * (y * z - w * x);
    o[8] = 2 * (x * z - w * y);     o[9] = 2 * (y * z + w * x);     o[10] = 1 - 2 * (x * x + y * y);
    o[3] = (real)P.p0[0] * (1 - u) + u * (real)P.p1[0];
    o[7] = (real)P.p0[1] * (1 - u) + u * (real)P.p1[1];
    o[11] = (real)P.p0[2] * (1 - u) + u * (real)P.p1[2];
    o[12] = 0; o[13] = 0; o[14] = 0; o[15] = 1;
    if (VEC) {
        store16<real>(T + row * 16, o); // 16-byte vector stores (the launcher has looked at the alignment)
    } else {
#pragma unroll
        for (int k = 0; k < 16; k++) T[row * 16 + k] = o[k];
    }
}

// rotation matrix (row-major 4x4) -> unit quaternion with s >= 0 (spatialmath r2q's convention)
void host_r2q(const double *T, double *q)
{
    const double R[3][3] = {{T[0], T[1], T[2]}, {T[4], T[5], T[6]}, {T[8], T[9], T[10]}};
    const double tr = R[0][0] + R[1][1] + R[2][2];
    if (tr > 0) {
        const double s = sqrt(tr + 1.0) * 2;
        q[0] = s / 4; q[1] = (R[2][1] - R[1][2]) / s; q[2] = (R[0][2] - R[2][0]) / s; q[3] = (R[1][0] - R[0][1]) / s;
    } else if (R[0][0] > R[1][1] && R[0][0] > R[2][2]) {
        const double s = sqrt(1.0 + R[0][0] - R[1][1] - R[2][2]) * 2;
        q[0] = (R[2][1] - R[1][2]) / s; q[1] = s / 4; q[2] = (R[0][1] + R[1][0]) / s; q[3] = (R[0][2] + R[2][0]) / s;
    } else if (R[1][1] > R[2][2]) {
        const double s = sqrt(1.0 + R[1][1] - R[0][0] - R[2][2]) * 2;
        q[0] = (R[0][2] - R[2][0]) / s; q[1] = (R[0][1] + R[1][0]) / s; q[2] = s / 4; q[3] = (R[1][2] + R[2][1]) / s;
    } else {
        const double s = sqrt(1.0 + R[2][2] - R[0][0] - R[1][1]) * 2;
        q[0] = (R[1][0] - R[0][1]) / s; q[1] = (R[0][2] + R[2][0]) / s; q[2] = (R[1][2] + R[2][1]) / s; q[3] = s / 4;
    }
    double nrm = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    if (q[0] < 0) nrm = -nrm;
    for (int k = 0; k < 4; k++) q[k] /= nrm;
}

// ---- mstraj sample table: pieces in row order; a piece is a quintic blend (jtraj with boundary velocities, sampled at
// t = (k + 1) dt) or a linear segment (q = (1 - s) q_prev + s q_next, s = t / tseg, t = t0 + k dt)
struct MsPiece {
    long long row0, rows;
    int kind;            // 0 quintic blend, 1 linear
    double tscal, t0, dt; // blend: tscal = blend duration; linear: tscal = tseg, t0 = first sample time
};

template <typename real>
__global__ void __launch_bounds__(256) k_mstraj(const MsPiece *__restrict__ pieces, const double *__restrict__ coef, int npieces, int n,
                                                long long nrows, real *__restrict__ q)
{
    const long long total = nrows * n;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        long long row; int j;
        split_elem(e, n, total, row, j);
        int lo = 0, hi = npieces - 1; // the piece that holds this row
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (pieces[mid].row0 <= row) lo = mid; else hi = mid - 1;
        }
        const MsPiece p = pieces[lo];
        const double *c = coef + ((size_t)lo * n + j) * 6;
        const double k = (double)(row - p.row0);
        double v;
        if (p.kind == 0) { // jtraj, trajectory.py:753-767: s = t / tscal, q = A s^5 + B s^4 + C s^3 + E s + F
            const double s = (k + 1) * p.dt / p.tscal;
            v = fma(fma(fma(fma(c[0], s, c[1]), s, c[2]) * s, s, c[3]), s, c[4]);
        } else {
            const double s = (p.t0 + k * p.dt) / p.tscal;
            v = (1 - s) * c[0] + s * c[1];
        }
        q[e] = (real)v;
    }
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

// ---- host side
// Every argument of the eight entry points is checked before any CUDA call, in one order: dtype, n (nmax = 0: the entry
// point takes none), N, the entry point's own scalar (bad_scalar: what is wrong with it), the host tables, then the
// device arrays -- non-NULL where required and N > 0, and aligned to their element size (es; 0: the dtype's) whenever
// they are passed.  ms: b2k_mstraj's piece table, which must hold at least one piece and cover the N rows in order.
// A rejection reads "<entry point>: bad arguments: <the argument and what is wrong with it>"; callers that match the
// "bad arguments" these functions have always reported keep working.
struct HostTable {
    const void *p;
    const char *name;
};
struct DevArray {
    const void *p;
    const char *name;
    bool required;
    unsigned es = 0;
};
struct MsTable {
    int npieces;
    const int64_t *row0, *rows;
    const int32_t *kind;
};

int pose_check(const char *fn, int dtype, int n, int nmax, long long N, const char *bad_scalar,
               std::initializer_list<HostTable> tables, std::initializer_list<DevArray> arrays, const MsTable *ms = nullptr)
{
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad arguments: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (nmax && (n < 1 || n > nmax)) { b2k_set_error("%s: bad arguments: n must be 1..%d, not %d", fn, nmax, n); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: bad arguments: N is negative", fn); return B2K_ERR_INVALID; }
    if (bad_scalar) { b2k_set_error("%s: bad arguments: %s", fn, bad_scalar); return B2K_ERR_INVALID; }
    for (const auto &t : tables)
        if (!t.p) { b2k_set_error("%s: bad arguments: %s is NULL", fn, t.name); return B2K_ERR_INVALID; }
    if (ms) {
        if (ms->npieces < 1) { b2k_set_error("%s: bad arguments: npieces must be at least 1", fn); return B2K_ERR_INVALID; }
        long long at = 0;
        for (int i = 0; i < ms->npieces; i++) {
            if (ms->row0[i] != at || ms->rows[i] < 0 || (ms->kind[i] != 0 && ms->kind[i] != 1)) { b2k_set_error("%s: bad arguments: piece %d is not contiguous / valid", fn, i); return B2K_ERR_INVALID; }
            at += ms->rows[i];
        }
        if (at != N) { b2k_set_error("%s: bad arguments: the pieces cover %lld rows, N = %lld", fn, at, N); return B2K_ERR_INVALID; }
    }
    for (const auto &x : arrays)
        if (x.required && N > 0 && !x.p) { b2k_set_error("%s: bad arguments: %s is NULL", fn, x.name); return B2K_ERR_INVALID; }
    for (const auto &x : arrays) {
        const unsigned es = x.es ? x.es : dtype == B2K_F64 ? 8u : 4u;
        if ((uintptr_t)x.p & (es - 1)) { b2k_set_error("%s: bad arguments: %s is not aligned to its element size (%u bytes)", fn, x.name, es); return B2K_ERR_INVALID; }
    }
    return B2K_OK;
}

// go(real(), std::bool_constant<VEC>()) for the call's dtype and VEC
template <typename F>
void by_dtype_vec(int dtype, bool vec, F &&go)
{
    if (dtype == B2K_F64) { if (vec) go(double(), std::true_type()); else go(double(), std::false_type()); }
    else { if (vec) go(float(), std::true_type()); else go(float(), std::false_type()); }
}

// the grid of the element-wise producers (one thread per (row, axis) element, grid-stride): at most 16 blocks per SM
unsigned elem_blocks(long long total) { return (unsigned)std::min((total + 255) / 256, 16LL * b2k_num_sms()); }

// counts the launch just made and reports its error, if any
int launched()
{
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

// The three pose-error entry points; servo: the output is v and arrived is required.
template <int ERR>
int pose_servo(const char *fn, bool servo, int dtype, const void *Te, const void *Tep, int64_t N, int64_t tep_stride,
               const double *gain, double threshold, void *out, int32_t *arrived, void *stream)
{
    if (int rc = pose_check(fn, dtype, 0, 0, N, tep_stride != 0 && tep_stride != 16 ? "tep_stride must be 0 (one target) or 16" : nullptr,
                            {}, {{Te, "Te", true}, {Tep, "Tep", true}, {out, servo ? "v" : "e", true}, {arrived, "arrived", servo, 4}}))
        return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(Te);
    double g[6];
    for (int k = 0; k < 6; k++) g[k] = gain ? gain[k] : 1.0;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)((N + 255) / 256);
    by_dtype_vec(dtype, (((uintptr_t)Te | (uintptr_t)Tep) & 15) == 0, [&](auto r, auto vec) {
        using real = decltype(r);
        k_pose_servo<real, decltype(vec)::value, ERR><<<blocks, 256, 0, st>>>((const real *)Te, (const real *)Tep, tep_stride, N,
                                                                              (real)g[0], (real)g[1], (real)g[2], (real)g[3], (real)g[4],
                                                                              (real)g[5], (real)threshold, (real *)out, arrived);
    });
    return launched();
}

} // namespace

extern "C" int b2k_angle_axis(int dtype, const void *Te, const void *Tep, int64_t N, int64_t tep_stride, void *e, void *stream)
{
    return pose_servo<ERR_ANGLE_AXIS>("b2k_angle_axis", false, dtype, Te, Tep, N, tep_stride, nullptr, 0.0, e, nullptr, stream);
}

extern "C" int b2k_p_servo(int dtype, const void *Te, const void *Tep, int64_t N, int64_t tep_stride, const double *gain,
                           double threshold, void *v, int32_t *arrived, void *stream)
{
    return pose_servo<ERR_ANGLE_AXIS>("b2k_p_servo", true, dtype, Te, Tep, N, tep_stride, gain, threshold, v, arrived, stream);
}

extern "C" int b2k_p_servo_rpy(int dtype, const void *Te, const void *Tep, int64_t N, int64_t tep_stride, const double *gain,
                               double threshold, void *v, int32_t *arrived, void *stream)
{
    return pose_servo<ERR_RPY_ZYX>("b2k_p_servo_rpy", true, dtype, Te, Tep, N, tep_stride, gain, threshold, v, arrived, stream);
}

extern "C" int b2k_jacob0_analytical(int dtype, int n, const void *T, const void *J, int64_t N, int representation, void *Ja,
                                     void *stream)
{
    if (int rc = pose_check("b2k_jacob0_analytical", dtype, n, B2K_MAX_JOINTS, N,
                            representation < 0 || representation > 3 ? "representation must be 0 rpy/xyz, 1 rpy/zyx, 2 eul, 3 exp" : nullptr,
                            {}, {{T, "T", true}, {J, "J", true}, {Ja, "Ja", true}}))
        return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(J);
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)((N + 63) / 64);
    const size_t smem = (size_t)2 * 32 * 6 * n * (dtype == B2K_F64 ? 8 : 4);
    by_dtype_vec(dtype, ((uintptr_t)T & 15) == 0, [&](auto r, auto vec) {
        using real = decltype(r);
        k_janalytical<real, decltype(vec)::value><<<blocks, 64, smem, st>>>((const real *)T, (const real *)J, N, n, representation, (real *)Ja);
    });
    return launched();
}

extern "C" int b2k_jtraj(int dtype, int n, const double *q0, const double *qf, const double *qd0, const double *qd1,
                         int64_t N, const void *t, double tscal, void *q, void *qd, void *qdd, void *stream)
{
    if (int rc = pose_check("b2k_jtraj", dtype, n, B2K_MAX_JOINTS, N, !(tscal > 0) ? "tscal must be positive" : nullptr,
                            {{q0, "q0"}, {qf, "qf"}}, {{t, "t", false}, {q, "q", true}, {qd, "qd", false}, {qdd, "qdd", false}}))
        return rc;
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
    const unsigned blocks = elem_blocks(N * n);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == B2K_F64)
        k_jtraj<double><<<blocks, 256, 0, st>>>(P, (const double *)t, N, (double *)q, (double *)qd, (double *)qdd);
    else
        k_jtraj<float><<<blocks, 256, 0, st>>>(P, (const float *)t, N, (float *)q, (float *)qd, (float *)qdd);
    return launched();
}

extern "C" int b2k_mtraj(int dtype, int kind, int n, const double *q0, const double *qf, const double *qd0, const double *qdf,
                         const double *V, int64_t N, const void *t, double tf, void *s, void *sd, void *sdd, double *tblend,
                         void *stream)
{
    const char *fn = "b2k_mtraj";
    if (int rc = pose_check(fn, dtype, n, B2K_MAX_JOINTS, N,
                            kind != 0 && kind != 1 ? "kind must be 0 (quintic) or 1 (trapezoidal)"
                            : !(tf > 0)            ? "tf must be positive (at least two samples)"
                                                   : nullptr,
                            {{q0, "q0"}, {qf, "qf"}}, {{t, "t", false}, {s, "s", true}, {sd, "sd", false}, {sdd, "sdd", false}}))
        return rc;
    MtrajP P;
    P.n = n;
    P.kind = kind;
    for (int j = 0; j < n; j++) {
        if (kind == 0) {
            if (!quintic_coeffs(q0[j], qf[j], tf, qd0 ? qd0[j] : 0.0, qdf ? qdf[j] : 0.0, P.c[j])) {
                b2k_set_error("%s: axis %d: singular boundary-condition system", fn, j);
                return B2K_ERR_INVALID;
            }
        } else { // trapezoidal_func, trajectory.py:552-565
            double v;
            if (!V || V[j] != V[j]) v = (qf[j] - q0[j]) / tf * 1.5; // NaN = not given
            else {
                const double d = qf[j] - q0[j];
                v = fabs(V[j]) * (d > 0 ? 1.0 : (d < 0 ? -1.0 : 0.0));
                if (fabs(v) < fabs(d) / tf) { b2k_set_error("%s: axis %d: V too small", fn, j); return B2K_ERR_INVALID; }
                if (fabs(v) > 2 * fabs(d) / tf) { b2k_set_error("%s: axis %d: V too big", fn, j); return B2K_ERR_INVALID; }
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
    const unsigned blocks = elem_blocks(N * n);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == B2K_F64)
        k_mtraj<double><<<blocks, 256, 0, st>>>(P, (const double *)t, N, (double *)s, (double *)sd, (double *)sdd);
    else
        k_mtraj<float><<<blocks, 256, 0, st>>>(P, (const float *)t, N, (float *)s, (float *)sd, (float *)sdd);
    return launched();
}

extern "C" int b2k_ctraj(int dtype, const double *T0, const double *T1, const void *s, int64_t N, void *T, void *stream)
{
    if (int rc = pose_check("b2k_ctraj", dtype, 0, 0, N, nullptr, {{T0, "T0"}, {T1, "T1"}}, {{s, "s", true}, {T, "T", true}}))
        return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(T);
    CtrajP P;
    host_r2q(T0, P.q0);
    host_r2q(T1, P.q1);
    double dot = 0;
    for (int k = 0; k < 4; k++) dot += P.q0[k] * P.q1[k];
    if (dot < 0) // shortest arc (qslerp: q0 = -q0)
        for (int k = 0; k < 4; k++) P.q0[k] = -P.q0[k];
    // the angle between the unit quaternions as 2 atan2(|q1 - q0|, |q1 + q0|): acos(dot) keeps only half the digits of
    // a small angle and is 0 below ~1e-8, where the orientation would then stay at T0's all the way and jump at s = 1
    double dm = 0, ds = 0;
    for (int k = 0; k < 4; k++) {
        dm += (P.q1[k] - P.q0[k]) * (P.q1[k] - P.q0[k]);
        ds += (P.q1[k] + P.q0[k]) * (P.q1[k] + P.q0[k]);
    }
    P.theta = 2 * atan2(sqrt(dm), sqrt(ds));
    P.sin_theta = sin(P.theta);
    P.lerp_only = !(fabs(P.theta) > 10 * 2.220446049250313e-16);
    for (int k = 0; k < 3; k++) { P.p0[k] = T0[4 * k + 3]; P.p1[k] = T1[4 * k + 3]; }
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)((N + 255) / 256);
    by_dtype_vec(dtype, ((uintptr_t)T & 15) == 0, [&](auto r, auto vec) {
        using real = decltype(r);
        k_ctraj<real, decltype(vec)::value><<<blocks, 256, 0, st>>>(P, (const real *)s, N, (real *)T);
    });
    return launched();
}

extern "C" int b2k_mstraj(int dtype, int n, int npieces, const int64_t *row0, const int64_t *rows, const int32_t *kind,
                          const double *tscal, const double *t0, const double *dt, const double *coef, int64_t N, void *q,
                          void *stream)
{
    const MsTable ms = {npieces, row0, rows, kind};
    if (int rc = pose_check("b2k_mstraj", dtype, n, B2K_MAX_QWIDTH, N, nullptr,
                            {{row0, "row0"}, {rows, "rows"}, {kind, "kind"}, {tscal, "tscal"}, {t0, "t0"}, {dt, "dt"}, {coef, "coef"}},
                            {{q, "q", true}}, &ms))
        return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(q);
    b2k_keep_mempool();
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<MsPiece> hp(npieces);
    for (int i = 0; i < npieces; i++) hp[i] = {row0[i], rows[i], kind[i], tscal[i], t0[i], dt[i]};
    MsPiece *dp = nullptr;
    double *dc = nullptr;
    const size_t cb = (size_t)npieces * n * 6 * sizeof(double);
    B2K_CUDA(cudaMallocAsync((void **)&dp, hp.size() * sizeof(MsPiece), st));
    B2K_CUDA(cudaMallocAsync((void **)&dc, cb, st));
    B2K_CUDA(cudaMemcpyAsync(dp, hp.data(), hp.size() * sizeof(MsPiece), cudaMemcpyHostToDevice, st));
    B2K_CUDA(cudaMemcpyAsync(dc, coef, cb, cudaMemcpyHostToDevice, st));
    B2K_CUDA(cudaStreamSynchronize(st)); // the host tables (hp, the caller's coef) may go away after this call returns
    const unsigned blocks = elem_blocks(N * n);
    if (dtype == B2K_F64) k_mstraj<double><<<blocks, 256, 0, st>>>(dp, dc, npieces, n, N, (double *)q);
    else k_mstraj<float><<<blocks, 256, 0, st>>>(dp, dc, npieces, n, N, (float *)q);
    const int rc = launched();
    cudaFreeAsync(dp, st);
    cudaFreeAsync(dc, st);
    return rc;
}
