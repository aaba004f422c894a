// b2k_ik.cuh -- batched Levenberg-Marquardt inverse kinematics, one fused persistent kernel (sm_90a).
//
// Replaces fknm.IK_LM_c (reference fknm.cpp:394-525 -> _IK_LM_Chan/_Wampler/_Sugihara
// ik.cpp:157-209 -> _IK_loop ik.cpp:19-75) and, with semantics = B2K_IK_SEM_PYTHON, the Python
// solver behind ETS.ikine_LM (IKSolver._solve IK.py:297-367 + IK_LM.step IK.py:994-1017).
//
// Mapping (DESIGN.md "Kernel K4"): one lane per IK problem, the whole LM loop in registers:
//   FK walk -> angle-axis error (ik.cpp:241-286) -> E = 1/2 e^T We e -> termination / wrap /
//   joint-limit test -> base-frame Jacobian -> g = J^T We e, A = J^T We J + Wn -> Cholesky
//   solve of the n x n SPD system (the reference forms A.inverse(), ik.cpp:171) -> q += dq.
// The kernel is persistent: the grid is sized to the machine and each lane pulls the next
// problem (grid-stride) as soon as its current one terminates, so lanes in a warp are always
// inside the same LM step code whatever iteration / search their problem is at.  Restarts
// draw q inside the joint limits from a counter-based generator keyed by (seed, row, search,
// joint) -- the reference uses unseeded libc rand() (ik.cpp:293) -- mirrored bit for bit by
// oracle/oracle_kin.c:orc_rand_u01 so the restart sequence is testable.
// Compute/latency-bound, not HBM-bound: per problem it reads 16 reals and writes n + 4 words.
#pragma once

#include "b2k_fkj.cuh"
#include <type_traits>

template <typename real, int N>
struct IkP {
    real qlim_l[N], qlim_h[N];
    real we[6];
    real ws[6]; // step weights of the pseudo-inverse solvers: 1 (NR) or sqrt(we) (GN)
    real lambda, tol;
    int ilimit, slimit, method, reject_jl, semantics, rng_per_row, has_q0, unit_w;
    unsigned long long seed;
};

__device__ __forceinline__ unsigned long long b2k_mix64(unsigned long long x)
{
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}

// uniform in [0,1): 53 random bits for fp64, the top 24 of the same word for fp32.
// Deliberately NOT inlined: a draw is ~60 instructions of 64-bit integer arithmetic per joint and happens once per
// search, but it used to be expanded at every place a problem can start or restart -- 5 000 of the 10 700
// instructions of k_ik_lm<float,7> -- and the LM evaluation (the only hot code) had to jump around it.
template <typename real>
__device__ __noinline__ real b2k_rand_u01(unsigned long long seed, unsigned long long row, unsigned search,
                                          unsigned joint)
{
    unsigned long long h = b2k_mix64(seed ^ (0x5851F42D4C957F2DULL * (row + 1)));
    h = b2k_mix64(h + (((unsigned long long)search << 32) | (unsigned long long)joint));
    if (sizeof(real) == 8) return (real)((double)(h >> 11) * (1.0 / 9007199254740992.0));
    return (real)((float)(h >> 40) * (1.0f / 16777216.0f));
}

template <typename real> __device__ __forceinline__ real b2k_sqrt(real x);
template <> __device__ __forceinline__ double b2k_sqrt<double>(double x) { return sqrt(x); }
template <> __device__ __forceinline__ float b2k_sqrt<float>(float x) { return sqrtf(x); }
template <typename real> __device__ __forceinline__ real b2k_atan2(real y, real x);
template <> __device__ __forceinline__ double b2k_atan2<double>(double y, double x) { return atan2(y, x); }
template <> __device__ __forceinline__ float b2k_atan2<float>(float y, float x) { return atan2f(y, x); }
// fmod runs once per joint when a search converges; out of line for the same reason as the draws (1 700 instructions)
static __device__ __noinline__ double b2k_fmod_out_of_line(double y, double x) { return fmod(y, x); }
static __device__ __noinline__ float b2k_fmod_out_of_line(float y, float x) { return fmodf(y, x); }
template <typename real> __device__ __forceinline__ real b2k_fmod(real y, real x) { return b2k_fmod_out_of_line(y, x); }
// 1 / sqrt(d) of a Cholesky pivot.  fp64 keeps the IEEE square root and division (the counters of the compiled
// reference are reproduced bit for bit on its fixtures, DESIGN 3.5); fp32 has no such contract (outcome tests, 1e-4
// bar) and takes the special-function unit's rsqrt: 1 instruction on the serial chain of the factorisation
// instead of ~20 with two slow-path branches.
template <typename real> __device__ __forceinline__ real b2k_rsqrt_pivot(real d);
template <> __device__ __forceinline__ double b2k_rsqrt_pivot<double>(double d) { return 1.0 / sqrt(d); }
template <> __device__ __forceinline__ float b2k_rsqrt_pivot<float>(float d) { return rsqrtf(d); }

// compile-time loop: the body receives std::integral_constant<int, I>, so every index into a register array is a
// constant expression.  (#pragma unroll left the triangular loops of the factorisation as run-time loops for two of
// the columns, which put the whole packed matrix in local memory: 22 LDL + 14 STL per evaluation on the serial chain.)
template <int B, int E, typename F>
__device__ __forceinline__ void b2k_static_for(F &&f)
{
    if constexpr (B < E) {
        f(std::integral_constant<int, B>());
        b2k_static_for<B + 1, E>(f);
    }
}

// restart sample, _rand_q ik.cpp:288-299: qlim_l + (U(-1,1) + 1) * range/2
template <typename real, int N>
__device__ __forceinline__ void ik_rand_q(const IkP<real, N> &K, unsigned long long row, unsigned search, real *q)
{
#pragma unroll
    for (int i = 0; i < N; i++) {
        real r = (real)2 * b2k_rand_u01<real>(K.seed, row, search, (unsigned)i) - (real)1;
        real range2 = (K.qlim_h[i] - K.qlim_l[i]) / (real)2;
        q[i] = (r + (real)1) * range2 + K.qlim_l[i];
    }
}

// angle-axis pose error, _angle_axis ik.cpp:241-286 (thresholds kept verbatim)
template <typename real>
__device__ __forceinline__ void ik_angle_axis(const Pose<real> &Te, const real *Tp /*12: row-major 3x4*/, real *e)
{
    e[0] = Tp[3] - Te.p[0];
    e[1] = Tp[7] - Te.p[1];
    e[2] = Tp[11] - Te.p[2];
    // R = Rep * Re^T ; R(i,j) = sum_k Rep(i,k) Re(j,k) ; Re(j,k) = column k, component j
    real R[3][3];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++)
            R[i][j] = Tp[i * 4 + 0] * Te.c0[j] + Tp[i * 4 + 1] * Te.c1[j] + Tp[i * 4 + 2] * Te.c2[j];
    real lx = R[2][1] - R[1][2], ly = R[0][2] - R[2][0], lz = R[1][0] - R[0][1];
    const real l2 = lx * lx + ly * ly + lz * lz;
    real ln, inv_ln = 0;
    if constexpr (sizeof(real) == 4) { // fp32: |l| and 1/|l| from one rsqrt (no IEEE sqrt + three divisions on the chain)
        inv_ln = rsqrtf(fmaxf(l2, 1e-30f));
        ln = l2 * inv_ln;
    } else {
        ln = b2k_sqrt<real>(l2);
    }
    real tr = R[0][0] + R[1][1] + R[2][2];
    if (ln < (real)1e-6) {
        if (tr > 0) {
            e[3] = e[4] = e[5] = 0;
        } else {
            const real pi2 = (real)1.57079632679489661923132169163975144;
            e[3] = pi2 * (R[0][0] + 1);
            e[4] = pi2 * (R[1][1] + 1);
            e[5] = pi2 * (R[2][2] + 1);
        }
    } else {
        real ang = b2k_atan2<real>(ln, tr - 1);
        if constexpr (sizeof(real) == 4) {
            const real sc = ang * inv_ln;
            e[3] = sc * lx; e[4] = sc * ly; e[5] = sc * lz;
        } else { // the reference's order of operations (ik.cpp:283-285)
            e[3] = ang * lx / ln;
            e[4] = ang * ly / ln;
            e[5] = ang * lz / ln;
        }
    }
}

// In-place Cholesky solve of the packed-lower SPD system A x = b (A: N(N+1)/2 entries, row-wise
// lower triangle).  Returns false on a non-positive / non-finite pivot.
template <typename real, int N>
__device__ __forceinline__ bool ik_chol_factor(real *A)
{ // in place: A <- L (row-wise packed lower triangle) with 1 / L_jj on the diagonal; false on a non-positive pivot
    bool ok = true;
    b2k_static_for<0, N>([&](auto jc) {
        constexpr int j = decltype(jc)::value, rj = j * (j + 1) / 2;
        real d = A[rj + j];
        b2k_static_for<0, j>([&](auto kc) { constexpr int k = decltype(kc)::value; d -= A[rj + k] * A[rj + k]; });
        ok = ok && (d > 0) && isfinite(d);
        const real inv = b2k_rsqrt_pivot<real>(d);
        A[rj + j] = inv; // store 1/L_jj
        b2k_static_for<j + 1, N>([&](auto ic) {
            constexpr int i = decltype(ic)::value, ri = i * (i + 1) / 2;
            real s = A[ri + j];
            b2k_static_for<0, j>([&](auto kc) { constexpr int k = decltype(kc)::value; s -= A[ri + k] * A[rj + k]; });
            A[ri + j] = s * inv;
        });
    });
    return ok;
}

template <typename real, int N>
__device__ __forceinline__ void ik_chol_subst(const real *A, real *b)
{ // b <- (L L^T)^-1 b for the factor ik_chol_factor left in A
    // forward L y = b
    b2k_static_for<0, N>([&](auto ic) {
        constexpr int i = decltype(ic)::value, ri = i * (i + 1) / 2;
        real s = b[i];
        b2k_static_for<0, i>([&](auto kc) { constexpr int k = decltype(kc)::value; s -= A[ri + k] * b[k]; });
        b[i] = s * A[ri + i];
    });
    // backward L^T x = y
    b2k_static_for<0, N>([&](auto ic) {
        constexpr int i = N - 1 - decltype(ic)::value;
        real s = b[i];
        b2k_static_for<i + 1, N>([&](auto kc) { constexpr int k = decltype(kc)::value; s -= A[k * (k + 1) / 2 + i] * b[k]; });
        b[i] = s * A[i * (i + 1) / 2 + i];
    });
}

template <typename real, int N>
__device__ __forceinline__ bool ik_chol_solve(real *A, real *b)
{
    const bool ok = ik_chol_factor<real, N>(A);
    ik_chol_subst<real, N>(A, b);
    return ok;
}

// ------------------------------------------------------------------ manipulability Jacobian pieces (ETS.jacobm, all six axes)
// For a 6 x N Jacobian (jx(a, k) = J[a, k]) with Gram matrix A = J J^T and Yoshikawa's m = sqrt(det A):
//   jacobm[i] = m * sum_{b,k} H_i[b,k] G[b,k],   G[:, k] = A^-1 J[:, k]   (A^-1 symmetric)
// k_jacobm_all (b2k_extra.cu) and the null-space term of the IK step below both use these two functions.
// b2k_gram_chol6: A = J J^T factorised in place by ik_chol_factor; returns m = prod L_aa (false: not factorisable;
// m and the factor are then inf / nan, as numpy's inv leaves them in the reference).
template <typename real, int N, typename JX>
__device__ __forceinline__ bool b2k_gram_chol6(JX jx, real *A, real &m)
{
#pragma unroll
    for (int a = 0; a < 6; a++)
#pragma unroll
        for (int b = 0; b <= a; b++) {
            real s = 0;
#pragma unroll
            for (int k = 0; k < N; k++) s = fma(jx(a, k), jx(b, k), s);
            A[a * (a + 1) / 2 + b] = s;
        }
    const bool ok = ik_chol_factor<real, 6>(A);
    m = 1;
#pragma unroll
    for (int a = 0; a < 6; a++) m *= A[a * (a + 1) / 2 + a]; // the diagonal holds 1 / L_aa
    m = (real)1 / m;
    return ok;
}

// H_i[r, k] of the Hessian (methods.cpp:16-32) formed from J on the fly.  Only for k >= i or r < 3: the angular rows
// below the diagonal are zero and the callers skip them.
template <typename real, typename JX>
__device__ __forceinline__ real b2k_hess_term(JX jx, int i, int r, int k)
{
    const int cc = r % 3, c1 = (cc + 1) % 3, c2 = (cc + 2) % 3, wrow = r < 3 ? 0 : 3;
    const int lo = k >= i ? i : k, hi = k >= i ? k : i;
    const real u1 = jx(3 + c1, lo), u2 = jx(3 + c2, lo);
    const real w1 = jx(wrow + c1, hi), w2 = jx(wrow + c2, hi);
    return fma(u1, w2, -(u2 * w1));
}

// acc[i] = sum_{b,k} H_i[b,k] G[b,k] for the factor A of J J^T that b2k_gram_chol6 left (jacobm[i] = m * acc[i]), from
// the unweighted base-frame J (J[k][a]).  G is streamed one column at a time (x = A^-1 J[:, k]) into the N sums instead
// of being held whole.
template <typename real, int N>
__device__ __forceinline__ void ik_jacobm_sums(const real (*J)[6], const real *A, real *acc)
{
    auto jx = [&](int a, int k) { return J[k][a]; };
#pragma unroll
    for (int i = 0; i < N; i++) acc[i] = 0;
#pragma unroll
    for (int k = 0; k < N; k++) {
        real x[6];
#pragma unroll
        for (int a = 0; a < 6; a++) x[a] = J[k][a];
        ik_chol_subst<real, 6>(A, x);
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int r = 0; r < 6; r++)
                if (k >= i || r < 3) acc[i] = fma(b2k_hess_term<real>(jx, i, r, k), x[r], acc[i]);
    }
}

// ------------------------------------------------------------------ null-space motion of the Python solver loop
// Reference IKSolver._calc_qnull / _null_Σ (restated in DESIGN (f-7)); host side: b2k_ikine_null.
//   qnull = (I - J^T (J J^T)^-1 J) g,   g = inv_kq sigma(q) + inv_km jacobm(q)
//   sigma_i = +((q_i - l_i) - pi_i)^2 / (ps - pi_i)^2   if q_i - l_i <= pi_i
//           = -((h_i - q_i) - pi_i)^2 / (ps - pi_i)^2   if h_i - q_i <= pi_i   (wins when both hold)
// use_q / use_m switch the terms (gain > 0 in the reference); inv_kq = 1 / kq, inv_km = 1 / km.
template <typename real, int N>
struct IkNs {
    real inv_kq, inv_km, ps;
    real pi[N];
    int use_q, use_m;
};

// qn <- qnull at q, from the unweighted base-frame J (J[k][a]).  The projector I - pinv(J) J is formed from the
// Cholesky factor of J J^T that the manipulability term needs anyway.  False when J J^T cannot be factorised (J has
// lost row rank): the caller abandons the search, as the step itself does at a singular normal matrix.
template <typename real, int N>
__device__ __forceinline__ bool ik_null_motion(const IkP<real, N> &K, const IkNs<real, N> &S, const real (*J)[6],
                                               const real *q, real *qn)
{
    auto jx = [&](int a, int k) { return J[k][a]; };
    real A[21], m;
    const bool ok = b2k_gram_chol6<real, N>(jx, A, m);
#pragma unroll
    for (int i = 0; i < N; i++) {
        real s = 0;
        if (S.use_q) {
            const real dl = q[i] - K.qlim_l[i], dh = K.qlim_h[i] - q[i], d = S.ps - S.pi[i];
            if (dh <= S.pi[i]) {
                const real t = dh - S.pi[i];
                s = -(t * t) / (d * d);
            } else if (dl <= S.pi[i]) {
                const real t = dl - S.pi[i];
                s = (t * t) / (d * d);
            }
            s *= S.inv_kq;
        }
        qn[i] = s;
    }
    if (S.use_m) {
        real acc[N];
        ik_jacobm_sums<real, N>(J, A, acc);
        const real c = S.inv_km * m;
#pragma unroll
        for (int i = 0; i < N; i++) qn[i] = fma(c, acc[i], qn[i]);
    }
    real y[6];
#pragma unroll
    for (int a = 0; a < 6; a++) {
        real s = 0;
#pragma unroll
        for (int k = 0; k < N; k++) s = fma(J[k][a], qn[k], s);
        y[a] = s;
    }
    ik_chol_subst<real, 6>(A, y);
#pragma unroll
    for (int k = 0; k < N; k++) {
        real s = qn[k];
#pragma unroll
        for (int a = 0; a < 6; a++) s = fma(-J[k][a], y[a], s);
        qn[k] = s;
    }
    return ok;
}

// ------------------------------------------------------------------ quadratic-programming step of the Python solver loop
// Reference IK_QP.step (restated in DESIGN (f-11)); host side: b2k_ikine_qp.  With x = (dq, s):
//   min 1/2 kj |dq|^2 + 1/2 w |s|^2 + c^T dq   s.t.  J dq + s = e,   w = ks / sum|e|,   c = -[km > 0] jacobm(q) / km
// and, with kq > 0, at most one velocity-damper row per joint (the upper one wins when both hold):
//   -dq_i <= inv_kq ((q_i - l_i) - ps) / (pi_i - ps)  if q_i - l_i <= pi_i
//    dq_i <= inv_kq ((h_i - q_i) - ps) / (pi_i - ps)  if h_i - q_i <= pi_i
// Eliminating s and dividing by w (w grows as e shrinks; fp32 needs the scaled form):
//   min 1/2 dq^T (lam I + J^T J) dq - r^T dq,   lam = (kj / ks) sum|e|,   r = J^T e + sum|e| / (km ks) jacobm(q)
// under one-sided bounds on single coordinates.  kj_ks = kj / ks, inv_kmks = 1 / (km ks), inv_kq = 1 / kq.
template <typename real, int N>
struct IkQp {
    real kj_ks, inv_kmks, inv_kq, ps;
    real pi[N];
    int use_q, use_m;
};

// dq of the step in g.  The bounded QP is a linear complementarity problem with the SPD matrix lam I + J^T J, solved by
// principal pivoting with the least-index rule (Murty), which terminates for such matrices: each round solves the
// equality problem with the current set of fixed coordinates -- their rows and columns replaced by identity rows, so
// every index stays static -- then frees the lowest-indexed fixed coordinate whose multiplier is negative, or fixes the
// lowest-indexed free one past its bound.  Without a damper row that is one Cholesky solve, the cost of an LM step.
// False (the search is abandoned) when a factorisation fails or the rounds run out; sum|e| = 0 gives dq = 0.
template <typename real, int N>
__device__ __forceinline__ bool ik_qp_step(const IkP<real, N> &K, const IkQp<real, N> &S, const real (*J)[6],
                                           const real *e, const real *q, real *g)
{
    real se = 0;
#pragma unroll
    for (int k = 0; k < 6; k++) se += fabs(e[k]);
    if (se == (real)0) {
#pragma unroll
        for (int i = 0; i < N; i++) g[i] = 0;
        return true;
    }
    const real lam = S.kj_ks * se;
    real r[N];
#pragma unroll
    for (int i = 0; i < N; i++) {
        real s = 0;
#pragma unroll
        for (int k = 0; k < 6; k++) s = fma(J[i][k], e[k], s);
        r[i] = s;
    }
    if constexpr (N >= 6) { // the host rejects km > 0 for fewer joints: J J^T is singular there
        if (S.use_m) {
            auto jx = [&](int a, int k) { return J[k][a]; };
            real A[21], m, acc[N];
            if (!b2k_gram_chol6<real, N>(jx, A, m)) return false;
            ik_jacobm_sums<real, N>(J, A, acc);
            const real cm = m * se * S.inv_kmks;
#pragma unroll
            for (int i = 0; i < N; i++) r[i] = fma(cm, acc[i], r[i]);
        }
    }
    // damper rows: bit i of `up` (dq_i <= bnd_i) or `lo` (dq_i >= bnd_i)
    unsigned up = 0, lo = 0;
    real bnd[N];
#pragma unroll
    for (int i = 0; i < N; i++) {
        bnd[i] = 0;
        if (S.use_q) {
            const real dl = q[i] - K.qlim_l[i], dh = K.qlim_h[i] - q[i], d = S.inv_kq / (S.pi[i] - S.ps);
            if (dh <= S.pi[i]) {
                up |= 1u << i;
                bnd[i] = (dh - S.ps) * d;
            } else if (dl <= S.pi[i]) {
                lo |= 1u << i;
                bnd[i] = -((dl - S.ps) * d);
            }
        }
    }
    const unsigned rows = up | lo;
    const real tol = (real)64 * (sizeof(real) == 8 ? (real)2.220446049250313e-16 : (real)1.1920929e-07);
    unsigned fixed = 0;
    for (int round = 0; round < 2 * N + 2; round++) {
        real A[N * (N + 1) / 2];
#pragma unroll
        for (int i = 0; i < N; i++) g[i] = ((fixed >> i) & 1u) ? bnd[i] : r[i];
#pragma unroll
        for (int i = 0; i < N; i++) {
            const bool fi = (fixed >> i) & 1u;
#pragma unroll
            for (int j = 0; j <= i; j++) {
                const bool fj = (fixed >> j) & 1u;
                real h = 0;
#pragma unroll
                for (int k = 0; k < 6; k++) h = fma(J[i][k], J[j][k], h);
                if (i == j) {
                    A[i * (i + 1) / 2 + j] = fi ? (real)1 : h + lam;
                } else {
                    A[i * (i + 1) / 2 + j] = (fi || fj) ? (real)0 : h;
                    if (fi && !fj) g[j] = fma(-h, bnd[i], g[j]);
                    if (fj && !fi) g[i] = fma(-h, bnd[j], g[i]);
                }
            }
        }
        if (!ik_chol_solve<real, N>(A, g)) return false;
        if (!rows) return true;
#pragma unroll
        for (int i = 0; i < N; i++)
            if ((fixed >> i) & 1u) g[i] = bnd[i];
        real Jx[6];
#pragma unroll
        for (int k = 0; k < 6; k++) {
            real s = 0;
#pragma unroll
            for (int j = 0; j < N; j++) s = fma(J[j][k], g[j], s);
            Jx[k] = s;
        }
        int pick = -1;
#pragma unroll
        for (int i = N - 1; i >= 0; i--) { // downwards: the lowest index that breaks a condition is picked
            if (!((rows >> i) & 1u)) continue;
            const real sg = ((up >> i) & 1u) ? (real)1 : (real)-1;
            if ((fixed >> i) & 1u) { // multiplier -sg * gradient must be >= 0
                real jj = 0;
#pragma unroll
                for (int k = 0; k < 6; k++) jj = fma(J[i][k], Jx[k], jj);
                const real lx = lam * g[i], grad = lx + jj - r[i];
                if (sg * grad > tol * (fabs(lx) + fabs(jj) + fabs(r[i]))) pick = i;
            } else if (sg * (g[i] - bnd[i]) > tol * (fabs(g[i]) + fabs(bnd[i]))) {
                pick = i;
            }
        }
        if (pick < 0) return true;
        fixed ^= 1u << pick;
    }
    return false;
}

// ------------------------------------------------------------------ one LM evaluation (+ update) in registers
// Evaluates the pose error e and cost E at q, then forms the Jacobian, the normal equations and the
// damped update dq (left in g).  Returns false when A cannot be factorised.
// (K.unit_w: We = I, the common case -- the weights are then left out of the 35 inner products)
// Pseudo-inverse update of the Newton-Raphson / Gauss-Newton solvers (STEP = 1), dq left in g:
//   NR (_IK_NR ik.cpp:121-155, _pseudo_inverse ik.cpp:211-224):  dq = V diag(s/(s^2+d^2)) U^T e
//   GN (_IK_GN ik.cpp:79-119): minimum-norm solution of (J^T We J) dq = J^T We e = pinv(We^1/2 J) We^1/2 e
// Both are  Jw^T (Jw Jw^T + d^2 I)^-1 ew  for n >= 6 (6x6 SPD, Cholesky) and
// (Jw^T Jw + d^2 I)^-1 Jw^T ew for n < 6 (n x n), Jw = diag(ws) J, ew = diag(ws) e -- the same operator
// as the reference's SVD wherever the factorisation exists; where it does not (a singular
// configuration with d = 0) the search is abandoned, where the reference takes a wild step.
// A mask that leaves fewer weighted rows than joints makes Jw^T Jw singular for every q, so such a step of n < 6
// joints takes the 6x6 row form too: with the masked rows decoupled it is the minimum-norm step whenever the
// weighted rows of J are independent.
template <typename real, int N>
__device__ __forceinline__ bool ik_pinv_step(const IkP<real, N> &K, real (*J)[6], const real *e, real *g)
{
    real ew[6];
    const real d2 = K.lambda * K.lambda;
    int wrows = 0; // rows the weights keep
#pragma unroll
    for (int a = 0; a < 6; a++) {
        ew[a] = K.ws[a] * e[a];
        wrows += K.ws[a] != (real)0 ? 1 : 0;
        if (!K.unit_w) {
#pragma unroll
            for (int j = 0; j < N; j++) J[j][a] *= K.ws[a];
        }
    }
    if (N >= 6 || wrows < N) {
        real A[21];
#pragma unroll
        for (int a = 0; a < 6; a++)
#pragma unroll
            for (int b = 0; b <= a; b++) {
                real s = (a == b) ? (d2 + (K.ws[a] == (real)0 ? (real)1 : (real)0)) : (real)0; // a masked row decouples
#pragma unroll
                for (int j = 0; j < N; j++) s = fma(J[j][a], J[j][b], s);
                A[a * (a + 1) / 2 + b] = s;
            }
        const bool ok = ik_chol_solve<real, 6>(A, ew);
#pragma unroll
        for (int j = 0; j < N; j++) {
            real s = 0;
#pragma unroll
            for (int a = 0; a < 6; a++) s = fma(J[j][a], ew[a], s);
            g[j] = s;
        }
        return ok;
    } else {
        real A[N * (N + 1) / 2];
#pragma unroll
        for (int i = 0; i < N; i++) {
            real s = 0;
#pragma unroll
            for (int a = 0; a < 6; a++) s = fma(J[i][a], ew[a], s);
            g[i] = s;
#pragma unroll
            for (int j = 0; j <= i; j++) {
                real t = (i == j) ? d2 : (real)0;
#pragma unroll
                for (int a = 0; a < 6; a++) t = fma(J[i][a], J[j][a], t);
                A[i * (i + 1) / 2 + j] = t;
            }
        }
        return ik_chol_solve<real, N>(A, g);
    }
}

// NS: add the null-space motion of IkNs S (Python semantics, N >= 7 only) to the update; S is unused otherwise.
// STEP = 2: the quadratic-programming step of IkQp S (Python semantics) instead of the LM step.
template <typename real, int N, int PROF, int STEP = 0, bool NS = false, typename XP = IkNs<real, N>>
__device__ __forceinline__ bool ik_eval(const ChainP<real, N> &P, const IkP<real, N> &K, const real *Tp, const real *q,
                                        real &Ecur, real *g, bool skip_step_if_converged,
                                        const XP *S = nullptr)
{
    Pose<real> Te;
    real zj[N][3], pj[N][3], e[6];
    // q holds the n joints in chain order whatever the chain's jindex (a sub-chain's jindices need not be 0..n-1): joint j
    // reads q[j], as q0, q_out and the joint limits are laid out (b2k_ik_lm)
    chain_forward<real, N, true, PROF, 1>(P, [&](int j, int) { return q[j]; }, Te, zj, pj);
    ik_angle_axis<real>(Te, Tp, e);
    real E = 0;
    if (K.unit_w) {
#pragma unroll
        for (int k = 0; k < 6; k++) E = fma(e[k], e[k], E);
    } else {
#pragma unroll
        for (int k = 0; k < 6; k++) E += e[k] * K.we[k] * e[k];
    }
    E *= (real)0.5;
    Ecur = E;
    if (skip_step_if_converged && E < K.tol) return true; // the C++ loop tests E before stepping (ik.cpp:48)
    real J[N][6];
#pragma unroll
    for (int j = 0; j < N; j++) {
        const bool rev = PROF == 1 ? true : (P.axis[j] < 3);
        if (rev) {
            real dx = Te.p[0] - pj[j][0], dy = Te.p[1] - pj[j][1], dz = Te.p[2] - pj[j][2];
            J[j][0] = fma(zj[j][1], dz, -(zj[j][2] * dy));
            J[j][1] = fma(zj[j][2], dx, -(zj[j][0] * dz));
            J[j][2] = fma(zj[j][0], dy, -(zj[j][1] * dx));
            J[j][3] = zj[j][0]; J[j][4] = zj[j][1]; J[j][5] = zj[j][2];
        } else {
            J[j][0] = zj[j][0]; J[j][1] = zj[j][1]; J[j][2] = zj[j][2];
            J[j][3] = 0; J[j][4] = 0; J[j][5] = 0;
        }
    }
    if constexpr (STEP == 2) return ik_qp_step<real, N>(K, *S, J, e, q, g);
    real qn[N];
    bool nok = true;
    if constexpr (NS) nok = ik_null_motion<real, N>(K, *S, J, q, qn); // before ik_pinv_step weighs J in place
    auto add_null = [&](bool ok) { // q += dq + qnull (IK_LM.step / IK_NR.step / IK_GN.step)
        if constexpr (NS) {
#pragma unroll
            for (int i = 0; i < N; i++) g[i] += qn[i];
            return ok && nok;
        }
        return ok;
    };
    if (STEP == 1) return add_null(ik_pinv_step<real, N>(K, J, e, g));
    const real wn = (K.method == B2K_LM_CHAN) ? K.lambda * E : (K.method == B2K_LM_WAMPLER) ? K.lambda : (E + K.lambda);
    real A[N * (N + 1) / 2];
    if (K.unit_w) {
#pragma unroll
        for (int i = 0; i < N; i++) {
            real s = 0;
#pragma unroll
            for (int k = 0; k < 6; k++) s = fma(J[i][k], e[k], s);
            g[i] = s;
#pragma unroll
            for (int j = 0; j <= i; j++) {
                real a = (i == j) ? wn : (real)0;
#pragma unroll
                for (int k = 0; k < 6; k++) a = fma(J[i][k], J[j][k], a);
                A[i * (i + 1) / 2 + j] = a;
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < N; i++) {
            real s = 0;
#pragma unroll
            for (int k = 0; k < 6; k++) s += J[i][k] * K.we[k] * e[k];
            g[i] = s;
#pragma unroll
            for (int j = 0; j <= i; j++) {
                real a = 0;
#pragma unroll
                for (int k = 0; k < 6; k++) a += J[i][k] * K.we[k] * J[j][k];
                A[i * (i + 1) / 2 + j] = a + (i == j ? wn : (real)0);
            }
        }
    }
    return add_null(ik_chol_solve<real, N>(A, g));
}

// wrap to [-pi, pi) the way each reference loop does, and test the joint limits
template <typename real, int N>
__device__ __forceinline__ bool ik_wrap_and_check(const IkP<real, N> &K, real *q)
{
    const real PI = (real)3.14159265358979323846264338327950288;
    bool inlim = true;
#pragma unroll
    for (int i = 0; i < N; i++) {
        if (K.semantics == B2K_IK_SEM_CPP) {
            q[i] = b2k_fmod<real>(q[i] + PI, (real)6.283185307179586) - PI; // ik.cpp:51: fmod keeps the dividend's sign
        } else {
            real w = b2k_fmod<real>(q[i] + PI, (real)2 * PI);
            if (w < 0) w += (real)2 * PI; // Python floor-modulo (IK.py:331)
            q[i] = w - PI;
        }
        inlim = inlim && !(q[i] < K.qlim_l[i] || q[i] > K.qlim_h[i]);
    }
    return inlim;
}

// ------------------------------------------------------------------ phase A: one lane per problem (flattened state machine)
// Every loop trip is exactly one LM evaluation for every active lane, whatever problem / search /
// iteration the lane is at, so the lanes of a warp never leave the common code.  With
// two_phase != 0 a lane does only the FIRST search of a problem; a problem whose first search
// fails is appended to the hard list (with its iteration contribution) for k_ik_restarts.
// Resident blocks per SM asked of ptxas: with the normal equations and the Jacobian in registers the fp32 kernels
// fit 128 registers (4 blocks) without spilling; the fp64 ones would take ~250 (2 blocks) and run 1-4 % faster held to 168 (3 blocks, ~150 B of spills)
// (DESIGN 3.5 has the sweep: 4 / 5 / 6 blocks measure the same, 8 spills and is 10 % slower).
template <typename real> constexpr int ik_min_blocks() { return sizeof(real) == 4 ? 4 : 3; }
// The kernels with the null-space term (k_ik_lm_ns, k_ik_restarts_ns) hold J, the Gram factor and the N Hessian sums
// at once.  Chosen from -Xptxas -v: fp32 fits 168 registers (3 blocks) without spilling up to N = 9 and 255 (2 blocks)
// at N = 10; fp64 at 255 (2 blocks) spills less than the plain fp64 k_ik_lm does at 168 (DESIGN (f-7) has the table).
template <typename real, int N> constexpr int ik_ns_min_blocks() { return sizeof(real) == 4 && N <= 9 ? 3 : 2; }

// The kernels with the quadratic-programming step (k_ik_lm_qp, k_ik_restarts_qp) hold J, the factor of the bounded
// system and, from N = 6, the Gram factor and the N Hessian sums.  Chosen from -Xptxas -v (DESIGN (f-11) has the table).
template <typename real, int N> constexpr int ik_qp_min_blocks() { return sizeof(real) == 4 && N <= 7 ? 3 : 2; }

// The bodies of the two kernels are shared by the plain kernels (k_ik_lm, k_ik_restarts), their null-space
// variants (k_ik_lm_ns, k_ik_restarts_ns, NS = true, S = their IkNs parameter) and the QP kernels (STEP = 2, S = their
// IkQp parameter); S is unused otherwise.
template <typename real, int N, int PROF, int STEP, bool NS, typename XP = IkNs<real, N>>
__device__ __forceinline__ void
ik_lm_body(const ChainP<real, N> &P, const IkP<real, N> &K, const std::enable_if_t<true, XP> *S,
           const real *__restrict__ Tep, const real *__restrict__ q0, long long nprob, real *__restrict__ q_out,
           int *__restrict__ success, int *__restrict__ iterations, int *__restrict__ searches,
           real *__restrict__ residual, int two_phase, int *__restrict__ hard_idx, int *__restrict__ hard_count,
           int iter_cap, const int *__restrict__ in_list, const int *__restrict__ in_count, int *__restrict__ cont_idx,
           int *__restrict__ cont_count)
{
    // Segmented first search (two_phase only): with iter_cap > 0 a problem that is still iterating after iter_cap
    // evaluations in THIS launch parks its state (q in q_out, the search's evaluation count in iterations) and is
    // appended to cont_idx; a later launch with in_list = that list resumes it.  Quick problems then never share a
    // warp with slow ones for long, and the slow ones are re-packed into full warps.
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long pos = (long long)blockIdx.x * blockDim.x + threadIdx.x; // position in the work list
    const long long nwork = in_list ? (long long)*in_count : nprob;
    const bool cpp = K.semantics == B2K_IK_SEM_CPP;

    real q[N], Tp[12], E = 0;
    int it = 0, search = 0, iter = 0; // search is 0-based here; reported 1-based (cpp: ik.cpp:39-69, python: IK.py:299-348)
    int evals = 0;                    // evaluations of the current problem in this launch
    long long idx = 0;
    // A lane asks for its next problem by setting `fetch`; the fetch itself (target load, first q) is expanded ONCE, at
    // the top of the loop, instead of at each of the nine places a problem can end -- the loop body is the LM
    // evaluation plus ~200 instructions of bookkeeping, and stays inside the instruction caches.
    bool fetch = true;
    pos -= stride;

    auto begin_problem = [&]() {
        const real *t = Tep + idx * 16;
#pragma unroll
        for (int k = 0; k < 12; k++) Tp[k] = t[k];
        const unsigned long long row = K.rng_per_row ? (unsigned long long)idx : 0ULL;
        evals = 0;
        E = 0; it = 0; search = 0;
        if (in_list) { // resume a parked first search
#pragma unroll
            for (int i = 0; i < N; i++) q[i] = q_out[idx * N + i];
            iter = iterations[idx];
            return;
        }
        if (K.has_q0) {
#pragma unroll
            for (int i = 0; i < N; i++) q[i] = q0[idx * N + i];
        } else {
            ik_rand_q<real, N>(K, row, 0u, q);
        }
        iter = cpp ? 1 : 0; // the C++ loop's first search starts counting at 1 (ik.cpp:39), later ones at 0 (ik.cpp:67)
    };
    auto next_problem = [&]() { fetch = true; };
    // park the running first search when this launch's evaluation budget for it is used up
    auto maybe_yield = [&]() {
        if (iter_cap > 0 && ++evals >= iter_cap) {
#pragma unroll
            for (int i = 0; i < N; i++) q_out[idx * N + i] = q[i];
            iterations[idx] = iter;
            cont_idx[atomicAdd(cont_count, 1)] = (int)idx;
            next_problem();
        }
    };
    auto finish = [&](int ok, int its, int srch) {
#pragma unroll
        for (int i = 0; i < N; i++) q_out[idx * N + i] = q[i];
        success[idx] = ok;
        iterations[idx] = its;
        searches[idx] = srch;
        residual[idx] = E;
        next_problem();
    };
    // this search failed with `iter` evaluations counted: restart, hand over to phase B, or give up
    auto search_failed = [&]() {
        it += iter; iter = 0; search++;
        const unsigned long long row = K.rng_per_row ? (unsigned long long)idx : 0ULL;
        if (search >= K.slimit) {
            if (cpp) ik_rand_q<real, N>(K, row, (unsigned)search, q); // ik.cpp:66-69: a fresh draw is what remains in q
            finish(0, it, cpp ? K.slimit + 1 : K.slimit);              // python: IK.py:360-367
            return;
        }
        if (two_phase) {
            iterations[idx] = it;
            hard_idx[atomicAdd(hard_count, 1)] = (int)idx;
            next_problem();
            return;
        }
        ik_rand_q<real, N>(K, row, (unsigned)search, q);
    };

    while (true) {
        if (fetch) {
            pos += stride;
            if (pos >= nwork) break;
            idx = in_list ? (long long)in_list[pos] : pos;
            begin_problem();
            fetch = false;
        }
        real g[N], Ecur;
        // one call site for both loop orders (the evaluation is ~600 instructions; two inlined copies only cost
        // instruction-cache misses): the C++ order skips the step when the test before it has already passed
        const bool ok = ik_eval<real, N, PROF, STEP, NS, XP>(P, K, Tp, q, Ecur, g, cpp, S);
        E = Ecur;
        if (cpp) {
            // test before stepping (ik.cpp:44-58)
            if (Ecur < K.tol) {
                const bool inlim = ik_wrap_and_check<real, N>(K, q);
                if (!K.reject_jl || inlim) finish(1, it + iter, search + 1);
                else search_failed(); // converged outside the limits: this search is abandoned
                continue;
            }
            iter++;
            if (ok) {
#pragma unroll
                for (int i = 0; i < N; i++) q[i] += g[i];
            }
            if (!ok || iter > K.ilimit) search_failed();
            else maybe_yield();
        } else {
            // count the step, apply it, then test the PRE-step E (IK.py:314-348)
            iter++;
            if (!ok) { search_failed(); continue; } // numpy LinAlgError: abandon the search (IK.py:321-324)
#pragma unroll
            for (int i = 0; i < N; i++) q[i] += g[i];
            if (Ecur < K.tol) {
                const bool inlim = ik_wrap_and_check<real, N>(K, q);
                if (inlim || !K.reject_jl) finish(1, it + iter, search + 1);
                else search_failed();
            } else if (iter >= K.ilimit) {
                search_failed();
            } else {
                maybe_yield();
            }
        }
    }
}

template <typename real, int N, int PROF, int STEP = 0>
__global__ void __launch_bounds__(B2K_THREADS, ik_min_blocks<real>())
k_ik_lm(const __grid_constant__ ChainP<real, N> P, const __grid_constant__ IkP<real, N> K,
        const real *__restrict__ Tep, const real *__restrict__ q0, long long nprob, real *__restrict__ q_out,
        int *__restrict__ success, int *__restrict__ iterations, int *__restrict__ searches,
        real *__restrict__ residual, int two_phase, int *__restrict__ hard_idx, int *__restrict__ hard_count,
        int iter_cap, const int *__restrict__ in_list, const int *__restrict__ in_count, int *__restrict__ cont_idx,
        int *__restrict__ cont_count)
{
    ik_lm_body<real, N, PROF, STEP, false>(P, K, nullptr, Tep, q0, nprob, q_out, success, iterations, searches, residual,
                                           two_phase, hard_idx, hard_count, iter_cap, in_list, in_count, cont_idx,
                                           cont_count);
}

template <typename real, int N, int PROF, int STEP>
__global__ void __launch_bounds__(B2K_THREADS, ik_ns_min_blocks<real, N>())
k_ik_lm_ns(const __grid_constant__ ChainP<real, N> P, const __grid_constant__ IkP<real, N> K,
           const real *__restrict__ Tep, const real *__restrict__ q0, long long nprob, real *__restrict__ q_out,
           int *__restrict__ success, int *__restrict__ iterations, int *__restrict__ searches,
           real *__restrict__ residual, int two_phase, int *__restrict__ hard_idx, int *__restrict__ hard_count,
           int iter_cap, const int *__restrict__ in_list, const int *__restrict__ in_count, int *__restrict__ cont_idx,
           int *__restrict__ cont_count, const __grid_constant__ IkNs<real, N> S)
{
    ik_lm_body<real, N, PROF, STEP, true>(P, K, &S, Tep, q0, nprob, q_out, success, iterations, searches, residual,
                                          two_phase, hard_idx, hard_count, iter_cap, in_list, in_count, cont_idx,
                                          cont_count);
}

template <typename real, int N, int PROF>
__global__ void __launch_bounds__(B2K_THREADS, ik_qp_min_blocks<real, N>())
k_ik_lm_qp(const __grid_constant__ ChainP<real, N> P, const __grid_constant__ IkP<real, N> K,
           const real *__restrict__ Tep, const real *__restrict__ q0, long long nprob, real *__restrict__ q_out,
           int *__restrict__ success, int *__restrict__ iterations, int *__restrict__ searches,
           real *__restrict__ residual, int two_phase, int *__restrict__ hard_idx, int *__restrict__ hard_count,
           int iter_cap, const int *__restrict__ in_list, const int *__restrict__ in_count, int *__restrict__ cont_idx,
           int *__restrict__ cont_count, const __grid_constant__ IkQp<real, N> S)
{
    ik_lm_body<real, N, PROF, 2, false, IkQp<real, N>>(P, K, &S, Tep, q0, nprob, q_out, success, iterations, searches, residual,
                                        two_phase, hard_idx, hard_count, iter_cap, in_list, in_count, cont_idx,
                                        cont_count);
}

// ------------------------------------------------------------------ phase B: G lanes per hard problem, searches in parallel
// The restart draws are counter-based (seed, row, search, joint), so search s of a problem does not
// depend on searches 0..s-1.  A group of G lanes therefore runs G consecutive searches of one hard
// problem at the same time; the lowest-numbered successful search wins and the iteration counter
// is the sum of the contributions of all lower-numbered searches plus its own -- exactly what
// the sequential loop reports, but the latency of a problem needing k restarts drops from
// k x ilimit LM iterations to ceil(k / G) x ilimit.
template <typename real, int N, int PROF, int G, int STEP, bool NS, typename XP = IkNs<real, N>>
__device__ __forceinline__ void
ik_restarts_body(const ChainP<real, N> &P, const IkP<real, N> &K, const std::enable_if_t<true, XP> *S,
                 const real *__restrict__ Tep, real *__restrict__ q_out, int *__restrict__ success,
                 int *__restrict__ iterations, int *__restrict__ searches, real *__restrict__ residual,
                 const int *__restrict__ hard_idx, const int *__restrict__ hard_count, int s_first, int max_batches,
                 int *__restrict__ out_idx, int *__restrict__ out_count)
{
    // s_first: first (0-based) search of this launch; max_batches: batches of G searches a problem may run here.
    // A problem still unsolved after max_batches batches is appended to out_idx (its iteration total parked in
    // iterations[]) for a later launch with a wider group -- most hard problems need one or two restarts, so a
    // narrow first round (G = 2) does a quarter of the work of running G = 8 searches for every one of them.
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int sub = lane % G, gbase = lane - sub;
    const bool cpp = K.semantics == B2K_IK_SEM_CPP;
    const long long ngroups = (long long)gridDim.x * (blockDim.x / G);
    const int nhard = *hard_count;
    for (long long h = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / G; ; h += ngroups) {
        // all lanes of a warp leave together (the loop below uses warp-wide shuffles)
        const long long h_first = h - (lane / G); // group 0's h in this warp
        if (h_first >= nhard) break;
        const bool have = h < nhard;
        const long long idx = have ? hard_idx[h] : 0;
        const unsigned long long row = K.rng_per_row ? (unsigned long long)idx : 0ULL;
        real Tp[12];
#pragma unroll
        for (int k = 0; k < 12; k++) Tp[k] = Tep[idx * 16 + k];
        int it_total = have ? iterations[idx] : 0;
        bool done = !have;
        int batches = 0;
        for (int s0 = s_first; s0 < K.slimit; s0 += G, batches++) { // batch of searches s0 .. s0+G-1 (0-based; search 0 was phase A)
            if (__all_sync(FULL, done)) break;
            if (batches >= max_batches) break;
            const int s = s0 + sub;
            const bool run = !done && s < K.slimit;
            real q[N], E = 0;
            int iters = 0;
            bool won = false;
            if (run) ik_rand_q<real, N>(K, row, (unsigned)s, q);
            bool going = run;
            while (__any_sync(FULL, going)) {
                if (going) {
                    real g[N], Ecur;
                    const bool ok = ik_eval<real, N, PROF, STEP, NS, XP>(P, K, Tp, q, Ecur, g, cpp, S);
                    E = Ecur;
                    if (cpp) {
                        if (Ecur < K.tol) {
                            const bool inlim = ik_wrap_and_check<real, N>(K, q);
                            won = !K.reject_jl || inlim;
                            going = false;
                        } else {
                            iters++;
                            if (ok) {
#pragma unroll
                                for (int i = 0; i < N; i++) q[i] += g[i];
                            }
                            if (!ok || iters > K.ilimit) going = false;
                        }
                    } else {
                        iters++;
                        if (!ok) going = false;
                        else {
#pragma unroll
                            for (int i = 0; i < N; i++) q[i] += g[i];
                            if (Ecur < K.tol) {
                                const bool inlim = ik_wrap_and_check<real, N>(K, q);
                                won = inlim || !K.reject_jl;
                                going = false;
                            } else if (iters >= K.ilimit) going = false;
                        }
                    }
                }
            }
            // group reduction: lowest successful search wins; iteration contributions of the searches before it add up
            const unsigned gmask = G >= 32 ? 0xffffffffu : ((1u << (G & 31)) - 1u);
            const unsigned wins = (__ballot_sync(FULL, won) >> gbase) & gmask;
            const int wsub = wins ? (__ffs(wins) - 1) : G;
            int pre = 0, all = 0; // sum of iters over subs < wsub / over the whole batch
#pragma unroll
            for (int k = 0; k < G; k++) {
                const int v = __shfl_sync(FULL, iters, gbase + k);
                all += v;
                if (k < wsub) pre += v;
            }
            if (!done) {
                if (wins) {
                    if (sub == wsub) {
#pragma unroll
                        for (int i = 0; i < N; i++) q_out[idx * N + i] = q[i];
                        success[idx] = 1;
                        iterations[idx] = it_total + pre + iters;
                        searches[idx] = s + 1;
                        residual[idx] = E;
                    }
                    done = true;
                } else {
                    it_total += all;
                    if (s0 + G >= K.slimit) { // every search failed: report like the sequential loops do
                        const int last = K.slimit - 1 - s0; // sub that ran the last search
                        if (sub == last) {
                            if (cpp) ik_rand_q<real, N>(K, row, (unsigned)K.slimit, q); // ik.cpp:69: a fresh draw is what remains in q
#pragma unroll
                            for (int i = 0; i < N; i++) q_out[idx * N + i] = q[i];
                            success[idx] = 0;
                            iterations[idx] = it_total;
                            searches[idx] = cpp ? K.slimit + 1 : K.slimit;
                            residual[idx] = E;
                        }
                        done = true;
                    }
                }
            }
        }
        if (!done && sub == 0 && out_idx) { // out of batches for this launch: hand the problem to the next round
            iterations[idx] = it_total;
            out_idx[atomicAdd(out_count, 1)] = (int)idx;
        }
    }
}

template <typename real, int N, int PROF, int G, int STEP = 0>
__global__ void __launch_bounds__(B2K_THREADS, ik_min_blocks<real>())
k_ik_restarts(const __grid_constant__ ChainP<real, N> P, const __grid_constant__ IkP<real, N> K,
              const real *__restrict__ Tep, real *__restrict__ q_out, int *__restrict__ success,
              int *__restrict__ iterations, int *__restrict__ searches, real *__restrict__ residual,
              const int *__restrict__ hard_idx, const int *__restrict__ hard_count, int s_first, int max_batches,
              int *__restrict__ out_idx, int *__restrict__ out_count)
{
    ik_restarts_body<real, N, PROF, G, STEP, false>(P, K, nullptr, Tep, q_out, success, iterations, searches, residual,
                                                    hard_idx, hard_count, s_first, max_batches, out_idx, out_count);
}

template <typename real, int N, int PROF, int G, int STEP>
__global__ void __launch_bounds__(B2K_THREADS, ik_ns_min_blocks<real, N>())
k_ik_restarts_ns(const __grid_constant__ ChainP<real, N> P, const __grid_constant__ IkP<real, N> K,
                 const real *__restrict__ Tep, real *__restrict__ q_out, int *__restrict__ success,
                 int *__restrict__ iterations, int *__restrict__ searches, real *__restrict__ residual,
                 const int *__restrict__ hard_idx, const int *__restrict__ hard_count, int s_first, int max_batches,
                 int *__restrict__ out_idx, int *__restrict__ out_count, const __grid_constant__ IkNs<real, N> S)
{
    ik_restarts_body<real, N, PROF, G, STEP, true>(P, K, &S, Tep, q_out, success, iterations, searches, residual,
                                                   hard_idx, hard_count, s_first, max_batches, out_idx, out_count);
}

template <typename real, int N, int PROF, int G>
__global__ void __launch_bounds__(B2K_THREADS, ik_qp_min_blocks<real, N>())
k_ik_restarts_qp(const __grid_constant__ ChainP<real, N> P, const __grid_constant__ IkP<real, N> K,
                 const real *__restrict__ Tep, real *__restrict__ q_out, int *__restrict__ success,
                 int *__restrict__ iterations, int *__restrict__ searches, real *__restrict__ residual,
                 const int *__restrict__ hard_idx, const int *__restrict__ hard_count, int s_first, int max_batches,
                 int *__restrict__ out_idx, int *__restrict__ out_count, const __grid_constant__ IkQp<real, N> S)
{
    ik_restarts_body<real, N, PROF, G, 2, false, IkQp<real, N>>(P, K, &S, Tep, q_out, success, iterations, searches, residual,
                                                 hard_idx, hard_count, s_first, max_batches, out_idx, out_count);
}

// kernel selection for ik_launch_n: the plain kernels, (NS) their null-space variants, or (STEP = 2) the QP kernels
template <typename real, int N, int PROF, int STEP, bool NS>
constexpr auto ik_kernel_a()
{
    if constexpr (STEP == 2) return &k_ik_lm_qp<real, N, PROF>;
    else if constexpr (NS) return &k_ik_lm_ns<real, N, PROF, STEP>;
    else return &k_ik_lm<real, N, PROF, STEP>;
}
template <typename real, int N, int PROF, int G, int STEP, bool NS>
constexpr auto ik_kernel_b()
{
    if constexpr (STEP == 2) return &k_ik_restarts_qp<real, N, PROF, G>;
    else if constexpr (NS) return &k_ik_restarts_ns<real, N, PROF, G, STEP>;
    else return &k_ik_restarts<real, N, PROF, G, STEP>;
}

template <typename real, int N, int STEP, bool NS>
int ik_launch_n(const b2k_chain_s *c, const IkArgs &a, cudaStream_t st)
{
    const real *Tep = (const real *)a.Tep, *q0 = (const real *)a.q0;
    real *q_out = (real *)a.q_out, *residual = (real *)a.residual;
    int *success = a.success, *iterations = a.iterations, *searches = a.searches;
    const long long nprob = a.N;
    const int ilimit = a.ilimit, slimit = a.slimit;
    ChainP<real, N> P;
    b2k_fill_chain<real, N>(c, nullptr, nullptr, true, P);
    IkP<real, N> K;
    for (int i = 0; i < N; i++) { K.qlim_l[i] = (real)c->qlim_l[i]; K.qlim_h[i] = (real)c->qlim_h[i]; }
    K.unit_w = 1;
    for (int k = 0; k < 6; k++) {
        K.we[k] = a.we ? (real)a.we[k] : (real)1;
        if (K.we[k] != (real)1) K.unit_w = 0;
        // NR weighs only the cost E, never the step (ik.cpp:141-146); GN weighs both (ik.cpp:102-103)
        K.ws[k] = (a.method == B2K_IK_GN && a.we) ? (real)sqrt(a.we[k] > 0 ? a.we[k] : 0.0) : (real)1;
    }
    K.lambda = (real)a.lambda; K.tol = (real)a.tol;
    K.ilimit = ilimit; K.slimit = slimit; K.method = a.method; K.reject_jl = a.reject_jl ? 1 : 0;
    K.semantics = a.semantics; K.rng_per_row = a.rng_per_row ? 1 : 0; K.has_q0 = q0 ? 1 : 0; K.seed = a.seed;
    const auto &gn = a.gains;
    std::conditional_t<STEP == 2, IkQp<real, N>, IkNs<real, N>> S{};
    if constexpr (STEP == 2) {
        S.use_q = gn.kq > 0 ? 1 : 0;
        S.use_m = gn.km > 0 ? 1 : 0;
        S.kj_ks = (real)(gn.kj / gn.ks);
        S.inv_kmks = S.use_m ? (real)(1.0 / (gn.km * gn.ks)) : (real)0;
        S.inv_kq = S.use_q ? (real)(1.0 / gn.kq) : (real)0;
        S.ps = (real)gn.ps;
        for (int i = 0; i < N; i++) S.pi[i] = S.use_q ? (real)gn.pi[i] : (real)0;
    } else if constexpr (NS) {
        S.use_q = gn.kq > 0 ? 1 : 0;
        S.use_m = gn.km > 0 ? 1 : 0;
        S.inv_kq = S.use_q ? (real)(1.0 / gn.kq) : (real)0; // the reference scales by 1.0 / λ (IK.py _calc_qnull)
        S.inv_km = S.use_m ? (real)(1.0 / gn.km) : (real)0;
        S.ps = (real)gn.ps;
        for (int i = 0; i < N; i++) S.pi[i] = (real)gn.pi[i];
    }
    // one launch of kern (NS, STEP = 2: with S appended as its last argument)
    auto go = [&](auto kern, long long grid, auto... args) {
        if constexpr (NS || STEP == 2) kern<<<(unsigned)grid, B2K_THREADS, 0, st>>>(args..., S);
        else kern<<<(unsigned)grid, B2K_THREADS, 0, st>>>(args...);
    };
    // Two phases when restarts are allowed and the batch is large enough to matter: phase A runs the
    // first search of every problem (one lane each); phase B runs the restarts of the problems that
    // failed it with B2K_IK_GROUP lanes per problem.  Scratch (hard list + counter) is stream-ordered.
    constexpr int G = 8;
    const bool two_phase = slimit > 1 && nprob >= 1024;
    // first search: with two phases, one problem per lane in two segments (IK_SEG1 evaluations, then the rest for the
    // problems still running); otherwise persistent lanes pulling problems
    constexpr int IK_SEG1 = 10;
    int *scratch = nullptr;
    if (two_phase) {
        b2k_keep_mempool(); // do not hand the pool's memory back to the OS at every synchronisation
        B2K_CUDA(cudaMallocAsync((void **)&scratch, sizeof(int) * (size_t)(2 * nprob + 4), st));
        B2K_CUDA(cudaMemsetAsync(scratch, 0, 4 * sizeof(int), st)); // one counter per list: no memset between the launches
    }
    // lists: hard (first search failed; phase A -> restart round one), parked (segment one -> two of the first search),
    // cont (round one -> two), third (round two -> three).  Two index buffers serve all four: the parked list is
    // consumed before round one writes `cont` into the same buffer, and the hard list before round two writes `third`.
    int *hard_count = scratch, *park_count = scratch ? scratch + 1 : nullptr, *cont_count = scratch ? scratch + 2 : nullptr;
    int *third_count = scratch ? scratch + 3 : nullptr;
    int *hard_idx = scratch ? scratch + 4 : nullptr, *cont_idx = scratch ? scratch + 4 + nprob : nullptr;
    auto launch_a = [&](auto kern) -> int {
        int per_sm = b2k_blocks_per_sm((const void *)kern, B2K_THREADS, 0);
        if (per_sm < 1) return per_sm < 0 ? per_sm : (b2k_set_error("ik kernel does not fit on an SM"), B2K_ERR_INVALID);
        long long grid = (long long)b2k_num_sms() * per_sm;
        long long need = (nprob + B2K_THREADS - 1) / B2K_THREADS;
        if (grid > need || two_phase) grid = need;
        if (grid < 1) grid = 1;
        const bool seg = two_phase && ilimit > IK_SEG1 + 2;
        go(kern, grid, P, K, Tep, q0, nprob, q_out, success, iterations, searches, residual, two_phase ? 1 : 0, hard_idx,
           hard_count, seg ? IK_SEG1 : 0, (const int *)nullptr, (const int *)nullptr, cont_idx, park_count);
        b2k_count_launch();
        B2K_CUDA(cudaGetLastError());
        if (seg) { // second segment: the parked problems, re-packed (the list length is only known on the device)
            go(kern, grid, P, K, Tep, q0, nprob, q_out, success, iterations, searches, residual, 1, hard_idx, hard_count, 0,
               (const int *)cont_idx, (const int *)park_count, (int *)nullptr, (int *)nullptr);
            b2k_count_launch();
            B2K_CUDA(cudaGetLastError());
        }
        return B2K_OK;
    };
    // restarts in two rounds: G = 4 lanes per hard problem for searches 1-4, then G = 8 for whatever is still unsolved
    auto launch_b = [&](auto kern, int g, const int *list, const int *count, int s_first, int max_batches, int *out_list,
                        int *out_cnt) -> int {
        int per_sm = b2k_blocks_per_sm((const void *)kern, B2K_THREADS, 0);
        if (per_sm < 1) return per_sm < 0 ? per_sm : (b2k_set_error("ik restart kernel does not fit on an SM"), B2K_ERR_INVALID);
        long long grid = (long long)b2k_num_sms() * per_sm;
        long long need = (nprob * g + B2K_THREADS - 1) / B2K_THREADS; // upper bound: every problem hard
        if (grid > need) grid = need;
        if (grid < 1) grid = 1;
        go(kern, grid, P, K, Tep, q_out, success, iterations, searches, residual, list, count, s_first, max_batches,
           out_list, out_cnt);
        b2k_count_launch();
        B2K_CUDA(cudaGetLastError());
        return B2K_OK;
    };
    // phase A, then (two phases) the restart rounds, on the kernels of the chain profile PROF
    auto launch_all = [&](auto prof) -> int {
        constexpr int PROF = decltype(prof)::value;
        const int rc = launch_a(ik_kernel_a<real, N, PROF, STEP, NS>());
        if (rc != B2K_OK || !two_phase) return rc;
        // Restart rounds: 4 lanes (searches 1-4), ONE batch of 8 lanes (searches 5-12), then whole warps (32 searches
        // per batch) for the handful of problems still unsolved -- a protocol whose hardest problem needs 50 (or all
        // 100) searches otherwise runs 6 (12) serial batches of 30 evaluations for a few dozen problems.  A search
        // limit too small for the earlier rounds starts with 8-lane groups, or keeps them to the end.
        constexpr int G1 = 4, G3 = 32;
        if (slimit <= 1 + G1)
            return launch_b(ik_kernel_b<real, N, PROF, G, STEP, NS>(), G, hard_idx, hard_count, 1, 0x7fffffff, nullptr, nullptr);
        const int rc1 = launch_b(ik_kernel_b<real, N, PROF, G1, STEP, NS>(), G1, hard_idx, hard_count, 1, 1, cont_idx, cont_count);
        if (rc1 != B2K_OK) return rc1;
        if (slimit <= 1 + G1 + G)
            return launch_b(ik_kernel_b<real, N, PROF, G, STEP, NS>(), G, cont_idx, cont_count, 1 + G1, 0x7fffffff, nullptr, nullptr);
        const int rc2 = launch_b(ik_kernel_b<real, N, PROF, G, STEP, NS>(), G, cont_idx, cont_count, 1 + G1, 1, hard_idx, third_count);
        if (rc2 != B2K_OK) return rc2;
        return launch_b(ik_kernel_b<real, N, PROF, G3, STEP, NS>(), G3, hard_idx, third_count, 1 + G1 + G, 0x7fffffff, nullptr, nullptr);
    };
    int rc = c->dh_like ? launch_all(std::integral_constant<int, 1>()) : launch_all(std::integral_constant<int, 0>());
    if (scratch) {
        cudaError_t e = cudaFreeAsync(scratch, st);
        if (e != cudaSuccess && rc == B2K_OK) rc = b2k_cuda_fail(e, "cudaFreeAsync");
    }
    return rc;
}

// The launcher of one translation unit (b2k_ik_*.cu): the kernels STEP and NS pick (ik_kernel_a / ik_kernel_b) at the
// chain's joint count.  The null-space kernels exist for 7..10 joints only: a full-rank J of a chain with n <= 6 has an
// empty null space, and b2k_ikine_null rejects such chains.
template <typename real, int STEP, bool NS = false>
int ik_launch(const b2k_chain_s *c, const IkArgs &a, cudaStream_t st)
{
    constexpr int NMIN = NS ? 7 : 1;
#define B2K_CASE(NN)                                                                                                   \
    case NN:                                                                                                           \
        if constexpr (NN >= NMIN) return ik_launch_n<real, NN, STEP, NS>(c, a, st);                                    \
        break;
    switch (c->n) {
        B2K_CASE(1) B2K_CASE(2) B2K_CASE(3) B2K_CASE(4) B2K_CASE(5)
        B2K_CASE(6) B2K_CASE(7) B2K_CASE(8) B2K_CASE(9) B2K_CASE(10)
    }
#undef B2K_CASE
    b2k_set_error("ik: unsupported joint count %d", c->n);
    return B2K_ERR_INVALID;
}
