// b2k_pose.cu -- batch producers / consumers either side of the kinematics path that work on poses
// (SURVEY 8f-2, 8f-3), one lane per row:
//   b2k_ctraj              Cartesian trajectory T0 -> T1 (tools/trajectory.py:782-841 -> SE3.interp: translation
//                          lerp + unit-quaternion slerp), the (N,4,4) batch is born in HBM where ik_LM consumes it
//   b2k_p_servo_rpy        tools/p_servo.py:46-106 with its default method="rpy": error in the end-effector frame,
//                          e = [t(Te^-1 Tep); tr2rpy(Te^-1 Tep, order="zyx")]
//   b2k_jacob0_analytical  ETS.jacob0_analytical (ETS.py:1570-1626): blkdiag(I, A^-1(Gamma(R))) J0 for the four
//                          rate representations rpy/xyz, rpy/zyx, eul (ZYZ), exp
//   b2k_mstraj             the sample table of tools/trajectory.py:852-1152 (multi-segment multi-axis trajectory):
//                          quintic blends and linear segments planned on the host, evaluated per (row, axis) here
// The angle conventions (tr2rpy, tr2eul, rotvelxform, quaternion slerp) belong to spatialmath-python, which is not
// part of the reference tree: they are restated from its documented definitions -- R = Rz(yaw) Ry(pitch) Rx(roll) for
// "zyx", R = Rx(yaw) Ry(pitch) Rz(roll) for "xyz", R = Rz(phi) Ry(theta) Rz(psi) for "eul", v = theta k for "exp" --
// and pinned by properties (tests: the analytical Jacobian equals the finite-difference derivative of Gamma(R(q));
// interpolation end points and constant angular rate), not by the package itself.
#include <math.h>

#include <vector>

#include "b2k_common.cuh"

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

// e = [Re^T (tp - te); rpy_zyx(Re^T Rep)], v = gain .* e, arrived = sum |e| < threshold
template <typename real, bool VEC>
__global__ void __launch_bounds__(256) k_servo_rpy(const real *__restrict__ Te, const real *__restrict__ Tep, long long tep_stride,
                                                   long long nrows, real g0, real g1, real g2, real g3, real g4, real g5,
                                                   real threshold, real *__restrict__ out, int *__restrict__ arrived)
{
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    // the three used rows of both poses: 16-byte vector loads where the arrays allow (the launcher looks)
    real a[12], b[12];
    if (VEC) {
        load12<real>(Te + row * 16, a);
        load12<real>(Tep + row * tep_stride, b);
    } else {
#pragma unroll
        for (int k = 0; k < 12; k++) { a[k] = Te[row * 16 + k]; b[k] = Tep[row * tep_stride + k]; }
    }
    real R[3][3], e[6];
    const real d[3] = {b[3] - a[3], b[7] - a[7], b[11] - a[11]};
#pragma unroll
    for (int i = 0; i < 3; i++) {
        e[i] = a[0 * 4 + i] * d[0] + a[1 * 4 + i] * d[1] + a[2 * 4 + i] * d[2];
#pragma unroll
        for (int j = 0; j < 3; j++) R[i][j] = a[0 * 4 + i] * b[0 * 4 + j] + a[1 * 4 + i] * b[1 * 4 + j] + a[2 * 4 + i] * b[2 * 4 + j];
    }
    rot_to_rpy_zyx<real>(R, e + 3);
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

} // namespace

extern "C" int b2k_jacob0_analytical(int dtype, int n, const void *T, const void *J, int64_t N, int representation, void *Ja,
                                     void *stream)
{
    const char *fn = "b2k_jacob0_analytical";
    if (n < 1 || n > B2K_MAX_JOINTS) { b2k_set_error("%s: n must be 1..%d", fn, B2K_MAX_JOINTS); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (representation < 0 || representation > 3) { b2k_set_error("%s: representation must be 0 rpy/xyz, 1 rpy/zyx, 2 eul, 3 exp", fn); return B2K_ERR_INVALID; }
    if (N < 0 || (N > 0 && (!T || !J || !Ja))) { b2k_set_error("%s: bad arguments", fn); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(J);
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)((N + 63) / 64);
    const bool vec = ((uintptr_t)T & 15) == 0;
    const size_t smem = (size_t)2 * 32 * 6 * n * (dtype == B2K_F64 ? 8 : 4);
    if (dtype == B2K_F64) {
        if (vec) k_janalytical<double, true><<<blocks, 64, smem, st>>>((const double *)T, (const double *)J, N, n, representation, (double *)Ja);
        else k_janalytical<double, false><<<blocks, 64, smem, st>>>((const double *)T, (const double *)J, N, n, representation, (double *)Ja);
    } else {
        if (vec) k_janalytical<float, true><<<blocks, 64, smem, st>>>((const float *)T, (const float *)J, N, n, representation, (float *)Ja);
        else k_janalytical<float, false><<<blocks, 64, smem, st>>>((const float *)T, (const float *)J, N, n, representation, (float *)Ja);
    }
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

extern "C" int b2k_p_servo_rpy(int dtype, const void *Te, const void *Tep, int64_t N, int64_t tep_stride, const double *gain,
                               double threshold, void *v, int32_t *arrived, void *stream)
{
    const char *fn = "b2k_p_servo_rpy";
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (N < 0 || (N > 0 && (!Te || !Tep || !v || !arrived))) { b2k_set_error("%s: bad arguments", fn); return B2K_ERR_INVALID; }
    if (tep_stride != 0 && tep_stride != 16) { b2k_set_error("%s: tep_stride must be 0 (one target) or 16", fn); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(Te);
    double g[6];
    for (int k = 0; k < 6; k++) g[k] = gain ? gain[k] : 1.0;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)((N + 255) / 256);
    const bool vec = (((uintptr_t)Te | (uintptr_t)Tep) & 15) == 0;
#define B2K_SR(REAL, V)                                                                                                        \
    k_servo_rpy<REAL, V><<<blocks, 256, 0, st>>>((const REAL *)Te, (const REAL *)Tep, tep_stride, N, (REAL)g[0], (REAL)g[1],  \
                                                 (REAL)g[2], (REAL)g[3], (REAL)g[4], (REAL)g[5], (REAL)threshold, (REAL *)v, arrived)
    if (dtype == B2K_F64) { if (vec) B2K_SR(double, true); else B2K_SR(double, false); }
    else { if (vec) B2K_SR(float, true); else B2K_SR(float, false); }
#undef B2K_SR
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

extern "C" int b2k_ctraj(int dtype, const double *T0, const double *T1, const void *s, int64_t N, void *T, void *stream)
{
    const char *fn = "b2k_ctraj";
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (!T0 || !T1) { b2k_set_error("%s: T0 / T1 is NULL", fn); return B2K_ERR_INVALID; }
    if (N < 0 || (N > 0 && (!s || !T))) { b2k_set_error("%s: bad arguments", fn); return B2K_ERR_INVALID; }
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
    const bool vec = ((uintptr_t)T & 15) == 0;
    if (dtype == B2K_F64) {
        if (vec) k_ctraj<double, true><<<blocks, 256, 0, st>>>(P, (const double *)s, N, (double *)T);
        else k_ctraj<double, false><<<blocks, 256, 0, st>>>(P, (const double *)s, N, (double *)T);
    } else {
        if (vec) k_ctraj<float, true><<<blocks, 256, 0, st>>>(P, (const float *)s, N, (float *)T);
        else k_ctraj<float, false><<<blocks, 256, 0, st>>>(P, (const float *)s, N, (float *)T);
    }
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

extern "C" int b2k_mstraj(int dtype, int n, int npieces, const int64_t *row0, const int64_t *rows, const int32_t *kind,
                          const double *tscal, const double *t0, const double *dt, const double *coef, int64_t N, void *q,
                          void *stream)
{
    const char *fn = "b2k_mstraj";
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (n < 1 || n > B2K_MAX_QWIDTH) { b2k_set_error("%s: n must be 1..%d", fn, B2K_MAX_QWIDTH); return B2K_ERR_INVALID; }
    if (npieces < 1 || !row0 || !rows || !kind || !tscal || !t0 || !dt || !coef) { b2k_set_error("%s: bad piece table", fn); return B2K_ERR_INVALID; }
    if (N < 0 || (N > 0 && !q)) { b2k_set_error("%s: bad N / q", fn); return B2K_ERR_INVALID; }
    long long at = 0;
    for (int i = 0; i < npieces; i++) {
        if (row0[i] != at || rows[i] < 0 || (kind[i] != 0 && kind[i] != 1)) { b2k_set_error("%s: piece %d is not contiguous / valid", fn, i); return B2K_ERR_INVALID; }
        at += rows[i];
    }
    if (at != N) { b2k_set_error("%s: the pieces cover %lld rows, N = %lld", fn, at, (long long)N); return B2K_ERR_INVALID; }
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
    long long blocks = (N * n + 255) / 256;
    const long long cap = (long long)b2k_num_sms() * 16;
    if (blocks > cap) blocks = cap;
    if (dtype == B2K_F64) k_mstraj<double><<<(unsigned)blocks, 256, 0, st>>>(dp, dc, npieces, n, N, (double *)q);
    else k_mstraj<float><<<(unsigned)blocks, 256, 0, st>>>(dp, dc, npieces, n, N, (float *)q);
    b2k_count_launch();
    cudaError_t e = cudaGetLastError();
    cudaFreeAsync(dp, st);
    cudaFreeAsync(dc, st);
    if (e != cudaSuccess) return b2k_cuda_fail(e, "k_mstraj launch");
    return B2K_OK;
}
