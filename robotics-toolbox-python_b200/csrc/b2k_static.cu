// b2k_static.cu -- static forces on a serial chain from one forward walk: the gravity load with the base-frame
// Jacobian (reference DynamicsMixin.gravjac), the joint torques of an end-effector wrench (pay) and the payload
// capacity under joint torque limits (paycap); plus the two elementwise helpers pay-from-J and joint friction.
//
// One lane walks one configuration, T = A_0 J_0(q) A_1 ... J_{n-1}(q) A_n (base folded into A_0, tool into A_n), and
// keeps per joint only its signed axis z_j and origin p_j (world frame) and, for the gravity load, one partial sum.
// With S_j = sum_{i>=j} m_i pc_i and M_j = sum_{i>=j} m_i (pc_i the COM of link i in the world frame), the gravity load
// of a revolute joint is
//     tau_j = -z_j . ((S_j - M_j p_j) x g) = (g x z_j) . (P_j + M_j p_j) - (g x z_j) . S,
// where P_j = sum_{i<j} m_i pc_i is the running prefix at joint j and S the total: the first term is formed during the
// walk, the second after it, so no second walk and no per-link COM storage.  A prismatic joint gives -M_j z_j . g.
// Frame-1 wrenches need the end-effector rotation, known only after the walk, which is why z_j and p_j are kept.
//
// Outputs are staged per warp in shared memory and written as the warp's contiguous block of rows.
#include "b2k_fkj.cuh"

enum : int { ST_GRAVJAC = 0, ST_PAY = 1, ST_PAYCAP = 2 };

#define B2K_STATIC_THREADS 64 // two warps: the fp64 n = 10 Jacobian stage (2 x 32 x 61 x 8 B) fits static shared memory

template <typename real, int N>
struct StaticP {
    real m[N];       // link masses
    real c[N][3];    // COM of link j in the frame right after joint j's elementary transform
    real msuf[N];    // sum_{i>=j} m_i
    real g[3];       // world-frame gravity (as the robot stores it, not negated)
    real tauR[N][2]; // paycap: column 0 the largest torque, column 1 the smallest
    int frame;       // 0: wrench in the world frame, 1: in the end-effector frame
};

// Stage K reals of every active lane's row (written by fill(st_row)) and store the warp's rows_here rows, which are
// contiguous in global memory, with consecutive lanes on consecutive elements.
template <typename real, int K, typename Fill>
__device__ __forceinline__ void stage_rows(real *st, int lane, bool active, int rows_here, real *gblock, Fill fill)
{
    constexpr int RS = K | 1; // odd row stride: the one-row-per-lane writes are conflict-free
    __syncwarp();
    if (active) fill(st + lane * RS);
    __syncwarp();
    const int total = rows_here * K;
    for (int e = lane; e < total; e += 32) {
        const int r = e / K;
        gblock[e] = st[r * RS + (e - r * K)];
    }
}

template <typename real, int N, int MODE>
__global__ void __launch_bounds__(B2K_STATIC_THREADS) k_static(const __grid_constant__ ChainP<real, N> P,
                                                               const __grid_constant__ StaticP<real, N> S,
                                                               const real *__restrict__ q, long long nrows, int ldq,
                                                               const real *__restrict__ w, int w_stride, real *__restrict__ tau,
                                                               real *__restrict__ J, int *__restrict__ joint)
{
    constexpr int STAGE = (MODE == ST_GRAVJAC ? 6 * N : N) | 1;
    __shared__ real stage[B2K_STATIC_THREADS / 32][32 * STAGE];
    const int lane = threadIdx.x & 31;
    const long long row0 = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31);
    if (row0 >= nrows) return; // whole warp past the end
    const long long row = row0 + lane;
    const bool active = row < nrows;
    const int rows_here = nrows - row0 < 32 ? (int)(nrows - row0) : 32;
    real *st = stage[threadIdx.x >> 5];
    const real *qr = q + (active ? row : row0) * ldq;

    real z[N][3], p[N][3], a[N];
    real s[3] = {0, 0, 0};
    Pose<real> T;
    pose_from_const(T, P.A[0]);
#pragma unroll
    for (int j = 0; j < N; j++) {
        if (j > 0) pose_mul_const_right(T, P.A[j], P.akind[j]);
        const int ax = P.axis[j];
        const real sg = P.flip[j] ? (real)-1 : (real)1;
        const int k = ax < 3 ? ax : ax - 3;
#pragma unroll
        for (int i = 0; i < 3; i++) {
            z[j][i] = sg * ((k == 0) ? T.c0[i] : (k == 1) ? T.c1[i] : T.c2[i]);
            p[j][i] = T.p[i];
        }
        pose_joint_right(T, ax, qr[P.jidx[j]] * sg, P.trig);
        if constexpr (MODE != ST_PAY) {
            if (ax < 3) { // (g x z_j) . (P_j + M_j p_j)
                const real h0 = S.g[1] * z[j][2] - S.g[2] * z[j][1];
                const real h1 = S.g[2] * z[j][0] - S.g[0] * z[j][2];
                const real h2 = S.g[0] * z[j][1] - S.g[1] * z[j][0];
                a[j] = h0 * fma(S.msuf[j], p[j][0], s[0]) + h1 * fma(S.msuf[j], p[j][1], s[1]) + h2 * fma(S.msuf[j], p[j][2], s[2]);
            } else {
                a[j] = -S.msuf[j] * (z[j][0] * S.g[0] + z[j][1] * S.g[1] + z[j][2] * S.g[2]);
            }
#pragma unroll
            for (int i = 0; i < 3; i++) {
                const real pc = fma(T.c0[i], S.c[j][0], fma(T.c1[i], S.c[j][1], fma(T.c2[i], S.c[j][2], T.p[i])));
                s[i] = fma(S.m[j], pc, s[i]);
            }
        }
    }
    pose_mul_const_right(T, P.A[N], P.akind[N]);

    real tg[N]; // gravity load
    if constexpr (MODE != ST_PAY) {
        const real u0 = s[1] * S.g[2] - s[2] * S.g[1]; // u = S x g; (g x z_j) . S = z_j . u
        const real u1 = s[2] * S.g[0] - s[0] * S.g[2];
        const real u2 = s[0] * S.g[1] - s[1] * S.g[0];
#pragma unroll
        for (int j = 0; j < N; j++) tg[j] = P.axis[j] < 3 ? a[j] - (z[j][0] * u0 + z[j][1] * u1 + z[j][2] * u2) : a[j];
    }
    if constexpr (MODE == ST_GRAVJAC) {
        stage_rows<real, N>(st, lane, active, rows_here, tau + row0 * N, [&](real *o) {
#pragma unroll
            for (int j = 0; j < N; j++) o[j] = tg[j];
        });
        stage_rows<real, 6 * N>(st, lane, active, rows_here, J + row0 * 6 * N, [&](real *o) {
#pragma unroll
            for (int j = 0; j < N; j++) {
                if (P.axis[j] < 3) {
                    const real dx = T.p[0] - p[j][0], dy = T.p[1] - p[j][1], dz = T.p[2] - p[j][2];
                    o[0 * N + j] = fma(z[j][1], dz, -(z[j][2] * dy));
                    o[1 * N + j] = fma(z[j][2], dx, -(z[j][0] * dz));
                    o[2 * N + j] = fma(z[j][0], dy, -(z[j][1] * dx));
                    o[3 * N + j] = z[j][0];
                    o[4 * N + j] = z[j][1];
                    o[5 * N + j] = z[j][2];
                } else {
                    o[0 * N + j] = z[j][0];
                    o[1 * N + j] = z[j][1];
                    o[2 * N + j] = z[j][2];
                    o[3 * N + j] = o[4 * N + j] = o[5 * N + j] = (real)0;
                }
            }
        });
        return;
    } else {
        // the wrench of this row, into the world frame
        const real *wr = w + (active ? row : row0) * w_stride;
        real f[3], mo[3];
#pragma unroll
        for (int i = 0; i < 3; i++) { f[i] = wr[i]; mo[i] = wr[3 + i]; }
        bool zero_w = false;
        if constexpr (MODE == ST_PAYCAP) { // unit wrench
            const real nn = f[0] * f[0] + f[1] * f[1] + f[2] * f[2] + mo[0] * mo[0] + mo[1] * mo[1] + mo[2] * mo[2];
            zero_w = !(nn > (real)0);
            const real inv = zero_w ? (real)0 : (real)1 / sqrt(nn);
#pragma unroll
            for (int i = 0; i < 3; i++) { f[i] *= inv; mo[i] *= inv; }
        }
        if (S.frame == 1) {
            real fw[3], mw[3];
#pragma unroll
            for (int i = 0; i < 3; i++) {
                fw[i] = fma(T.c0[i], f[0], fma(T.c1[i], f[1], T.c2[i] * f[2]));
                mw[i] = fma(T.c0[i], mo[0], fma(T.c1[i], mo[1], T.c2[i] * mo[2]));
            }
#pragma unroll
            for (int i = 0; i < 3; i++) { f[i] = fw[i]; mo[i] = mw[i]; }
        }
        real tp[N]; // -J0^T W
#pragma unroll
        for (int j = 0; j < N; j++) {
            if (P.axis[j] < 3) { // z . ((pe - p_j) x f + m)
                const real dx = T.p[0] - p[j][0], dy = T.p[1] - p[j][1], dz = T.p[2] - p[j][2];
                const real v0 = fma(dy, f[2], -(dz * f[1])) + mo[0];
                const real v1 = fma(dz, f[0], -(dx * f[2])) + mo[1];
                const real v2 = fma(dx, f[1], -(dy * f[0])) + mo[2];
                tp[j] = -(z[j][0] * v0 + z[j][1] * v1 + z[j][2] * v2);
            } else {
                tp[j] = -(z[j][0] * f[0] + z[j][1] * f[1] + z[j][2] * f[2]);
            }
        }
        if constexpr (MODE == ST_PAY) {
            stage_rows<real, N>(st, lane, active, rows_here, tau + row0 * N, [&](real *o) {
#pragma unroll
                for (int j = 0; j < N; j++) o[j] = tp[j];
            });
        } else {
            real wm[N];
            int arg = zero_w ? -1 : 0;
            real best = (real)INFINITY;
#pragma unroll
            for (int j = 0; j < N; j++) {
                const real lim = tp[j] > (real)0 ? S.tauR[j][0] : S.tauR[j][1];
                wm[j] = zero_w ? (real)NAN : (tp[j] == (real)0 ? (real)INFINITY : (lim - tg[j]) / tp[j]);
                if (!zero_w && wm[j] < best) { best = wm[j]; arg = j; } // first index on ties
            }
            stage_rows<real, N>(st, lane, active, rows_here, tau + row0 * N, [&](real *o) {
#pragma unroll
                for (int j = 0; j < N; j++) o[j] = wm[j];
            });
            if (active) joint[row] = arg;
        }
    }
}

// tau = -J^T W from a given J (N, 6, n): one thread per element of tau
template <typename real>
__global__ void __launch_bounds__(256) k_pay_j(const real *__restrict__ J, const real *__restrict__ W, int w_stride, int n,
                                               long long total, real *__restrict__ tau)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    long long row;
    int j;
    split_elem(e, n, total, row, j);
    const real *Jr = J + row * 6 * n + j;
    const real *Wr = W + row * w_stride;
    real t = Jr[0] * Wr[0];
#pragma unroll
    for (int k = 1; k < 6; k++) t = fma(Jr[(long long)k * n], Wr[k], t);
    tau[e] = -t;
}

// joint friction: tau = -(G^2 B qd + |G| Tc(qd)), the actuator terms rne adds (ne.c, SURVEY Appendix D.6)
template <typename real>
struct FrictionP {
    real gb[B2K_MAX_JOINTS];  // G^2 B
    real ag[B2K_MAX_JOINTS];  // |G|
    real tcp[B2K_MAX_JOINTS]; // Tc+
    real tcm[B2K_MAX_JOINTS]; // Tc-
};

template <typename real>
__global__ void __launch_bounds__(256) k_friction(const __grid_constant__ FrictionP<real> F, const real *__restrict__ qd, int n,
                                                  long long total, real *__restrict__ tau)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    long long row;
    int j;
    split_elem(e, n, total, row, j);
    const real v = qd[e];
    const real tc = v > (real)0 ? F.tcp[j] : (v < (real)0 ? F.tcm[j] : (real)0);
    tau[e] = -(F.gb[j] * v + F.ag[j] * tc);
}

// ------------------------------------------------------------------ host side
// One call of b2k_gravjac (mass, grav; tau = taug, J = J0), b2k_pay (w, w_stride, frame; tau) or b2k_paycap (mass, grav,
// w, w_stride, frame, tauR; tau = wmax, joint), as passed; what the mode does not read is NULL or 0.
struct StaticArgs {
    const void *q;
    long long nrows, ldq;
    const double *mass, *grav;
    const void *w;
    long long w_stride;
    int frame;
    const double *tauR;
    void *tau, *J;
    int *joint;
};

template <typename real, int N, int MODE>
static int static_launch_n(const b2k_chain_s *c, const StaticArgs &a, cudaStream_t st)
{
    ChainP<real, N> P;
    b2k_fill_chain<real, N>(c, nullptr, nullptr, true, P);
    StaticP<real, N> S;
    double suf = 0.0;
    for (int j = N - 1; j >= 0; j--) {
        const double *mj = a.mass ? a.mass + 4 * j : nullptr;
        S.m[j] = mj ? (real)mj[0] : (real)0;
        for (int i = 0; i < 3; i++) S.c[j][i] = mj ? (real)mj[1 + i] : (real)0;
        suf += mj ? mj[0] : 0.0;
        S.msuf[j] = (real)suf;
        S.tauR[j][0] = a.tauR ? (real)a.tauR[2 * j] : (real)0;
        S.tauR[j][1] = a.tauR ? (real)a.tauR[2 * j + 1] : (real)0;
    }
    for (int i = 0; i < 3; i++) S.g[i] = a.grav ? (real)a.grav[i] : (real)0;
    S.frame = a.frame;
    const unsigned blocks = (unsigned)((a.nrows + B2K_STATIC_THREADS - 1) / B2K_STATIC_THREADS);
    k_static<real, N, MODE><<<blocks, B2K_STATIC_THREADS, 0, st>>>(P, S, (const real *)a.q, a.nrows, (int)a.ldq, (const real *)a.w,
                                                                 (int)a.w_stride, (real *)a.tau, (real *)a.J, a.joint);
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

static int check_mass(const char *fn, const b2k_chain_s *c, const double *mass, const double *grav)
{
    if (!mass) { b2k_set_error("%s: mass table is NULL", fn); return B2K_ERR_INVALID; }
    if (!grav) { b2k_set_error("%s: grav is NULL", fn); return B2K_ERR_INVALID; }
    for (int j = 0; j < c->n; j++)
        for (int k = 0; k < 4; k++)
            if (!isfinite(mass[4 * j + k])) { b2k_set_error("%s: mass table entry (%d, %d) is not finite", fn, j, k); return B2K_ERR_INVALID; }
    return B2K_OK;
}

static int check_w_stride(const char *fn, int64_t w_stride)
{
    if (w_stride != 0 && w_stride != 6) { b2k_set_error("%s: w_stride must be 0 (one wrench) or 6 (one per row)", fn); return B2K_ERR_INVALID; }
    return B2K_OK;
}

// Every argument is checked before any CUDA call: the chain, then the host tables and scalars the mode reads, then the
// device arrays, each aligned to its element size.
template <int MODE>
static int static_dispatch(const char *fn, b2k_chain_t c, int dtype, const StaticArgs &a, void *stream)
{
    const bool mass = MODE != ST_PAY, wrench = MODE != ST_GRAVJAC;
    int rc;
    if ((rc = b2k_check_chain(fn, c, dtype, a.q, a.nrows, a.ldq))) return rc;
    if (mass && (rc = check_mass(fn, c, a.mass, a.grav))) return rc;
    if (wrench) {
        if ((rc = check_w_stride(fn, a.w_stride))) return rc;
        if (a.frame != 0 && a.frame != 1) { b2k_set_error("%s: frame must be 0 (world) or 1 (end effector)", fn); return B2K_ERR_INVALID; }
    }
    if (MODE == ST_PAYCAP && !a.tauR) { b2k_set_error("%s: tauR is NULL", fn); return B2K_ERR_INVALID; }
    const unsigned es = dtype == B2K_F64 ? 8 : 4;
    const long long N = a.nrows;
    if ((wrench && (rc = b2k_check_array(fn, MODE == ST_PAY ? "W" : "w", a.w, N, es))) ||
        (rc = b2k_check_array(fn, MODE == ST_GRAVJAC ? "taug" : MODE == ST_PAY ? "tau" : "wmax", a.tau, N, es)) ||
        (MODE == ST_GRAVJAC && (rc = b2k_check_array(fn, "J0", a.J, N, es))) ||
        (MODE == ST_PAYCAP && (rc = b2k_check_array(fn, "joint", a.joint, N, 4))))
        return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(a.q);
    cudaStream_t st = (cudaStream_t)stream;
    return b2k_for_joints(c->n, [&](auto n) {
        return dtype == B2K_F64 ? static_launch_n<double, n.value, MODE>(c, a, st) : static_launch_n<float, n.value, MODE>(c, a, st);
    });
}

extern "C" int b2k_gravjac(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *mass, const double *grav,
                           void *taug, void *J0, void *stream)
{
    return static_dispatch<ST_GRAVJAC>("b2k_gravjac", c, dtype, {q, N, ldq, mass, grav, nullptr, 0, 0, nullptr, taug, J0, nullptr},
                                       stream);
}

extern "C" int b2k_pay(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const void *W, int64_t w_stride, int frame,
                       void *tau, void *stream)
{
    return static_dispatch<ST_PAY>("b2k_pay", c, dtype, {q, N, ldq, nullptr, nullptr, W, w_stride, frame, nullptr, tau, nullptr, nullptr},
                                   stream);
}

extern "C" int b2k_paycap(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *mass, const double *grav,
                          const void *w, int64_t w_stride, int frame, const double *tauR, void *wmax, int32_t *joint, void *stream)
{
    return static_dispatch<ST_PAYCAP>("b2k_paycap", c, dtype, {q, N, ldq, mass, grav, w, w_stride, frame, tauR, wmax, nullptr, joint},
                                      stream);
}

extern "C" int b2k_pay_jacobian(int dtype, int n, const void *J, const void *W, int64_t w_stride, int64_t N, void *tau, void *stream)
{
    const char *fn = "b2k_pay_jacobian";
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (n < 1 || n > B2K_MAX_JOINTS) { b2k_set_error("%s: n = %d outside [1, %d]", fn, n, B2K_MAX_JOINTS); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: N is negative", fn); return B2K_ERR_INVALID; }
    const unsigned es = dtype == B2K_F64 ? 8 : 4;
    int rc;
    if ((rc = check_w_stride(fn, w_stride)) || (rc = b2k_check_array(fn, "J", J, N, es)) ||
        (rc = b2k_check_array(fn, "W", W, N, es)) || (rc = b2k_check_array(fn, "tau", tau, N, es)))
        return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(J);
    const long long total = (long long)N * n;
    const unsigned blocks = (unsigned)((total + 255) / 256);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == B2K_F64) k_pay_j<double><<<blocks, 256, 0, st>>>((const double *)J, (const double *)W, (int)w_stride, n, total, (double *)tau);
    else k_pay_j<float><<<blocks, 256, 0, st>>>((const float *)J, (const float *)W, (int)w_stride, n, total, (float *)tau);
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

template <typename real>
static int friction_launch(int n, const double *params, const real *qd, long long total, real *tau, cudaStream_t st)
{
    FrictionP<real> F = {};
    for (int j = 0; j < n; j++) {
        const double B = params[4 * j], G = params[4 * j + 1];
        F.gb[j] = (real)(G * G * B);
        F.ag[j] = (real)fabs(G);
        F.tcp[j] = (real)params[4 * j + 2];
        F.tcm[j] = (real)params[4 * j + 3];
    }
    k_friction<real><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(F, qd, n, total, tau);
    b2k_count_launch();
    B2K_CUDA(cudaGetLastError());
    return B2K_OK;
}

extern "C" int b2k_friction(int dtype, int n, const double *params, const void *qd, int64_t N, void *tau, void *stream)
{
    const char *fn = "b2k_friction";
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (n < 1 || n > B2K_MAX_JOINTS) { b2k_set_error("%s: n = %d outside [1, %d]", fn, n, B2K_MAX_JOINTS); return B2K_ERR_INVALID; }
    if (!params) { b2k_set_error("%s: params is NULL", fn); return B2K_ERR_INVALID; }
    for (int k = 0; k < 4 * n; k++)
        if (!isfinite(params[k])) { b2k_set_error("%s: params[%d] is not finite", fn, k); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: N is negative", fn); return B2K_ERR_INVALID; }
    const unsigned es = dtype == B2K_F64 ? 8 : 4;
    int rc;
    if ((rc = b2k_check_array(fn, "qd", qd, N, es)) || (rc = b2k_check_array(fn, "tau", tau, N, es))) return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(qd);
    const long long total = (long long)N * n;
    cudaStream_t st = (cudaStream_t)stream;
    return dtype == B2K_F64 ? friction_launch<double>(n, params, (const double *)qd, total, (double *)tau, st)
                            : friction_launch<float>(n, params, (const float *)qd, total, (float *)tau, st);
}
