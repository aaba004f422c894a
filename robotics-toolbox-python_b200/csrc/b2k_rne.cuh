// b2k_rne.cuh -- batched recursive Newton-Euler inverse dynamics for DH / MDH arms (sm_90a).
//
// Replaces the per-row frne.frne loop of DHRobot.rne (reference DHRobot.py:1442-1451 ->
// frne.c:106-230 -> newton_euler ne.c:62-492, rot_mat frne.c:310-351).
//
// Mapping (DESIGN.md "Kernel K3"): like the FK kernel, a warp owns a tile of 32 rows.  The
// (q, qd, qdd) tiles are loaded with coalesced 8-byte-granule loads into a per-warp smem stage
// and stay there for both recursions; lane l runs the Luh-Walker-Paul recursion for row l in
// registers with all link constants (sin/cos(alpha), a, d, m, r, I, G^2 Jm, ...) coming from
// the constant bank (kernel parameter struct).  The forward recursion keeps only what the
// backward one needs per link: F_j = m a_c, N_j = I wd + w x (I w), sin/cos(theta_j).  tau is
// staged and written back coalesced.  HBM-bound: 4n reals per row (192 B for Puma560 fp64).
//
// The arithmetic mirrors ne.c operation by operation (including its quirks for a prismatic
// first joint under modified DH, ne.c:187-204) so results track the reference to rounding.
#pragma once

#include "b2k_fkj.cuh"

template <typename real, int N>
struct RneP {
    // per link
    real sa[N], ca[N]; // sin/cos(alpha) evaluated on the host with libm, as frne.c:325-326 does per call
    real A[N], D[N], st0[N], ct0[N], offset[N];
    real m[N], r[N][3], I[N][9];
    real c_jm[N];  // G*G*Jm
    real c_b[N];   // G*G*B
    real c_tcp[N]; // |G|*Tc+
    real c_tcm[N]; // |G|*Tc-
    int prismatic[N];
    real psrc[N][3]; // p* + r (standard DH backward recursion, ne.c:415-417), summed on the host
    real ps[N][3]; // p* of a revolute link: (a, d sin(alpha), d cos(alpha)) for DH, (a, -d sin(alpha), d cos(alpha)) for MDH
    real grav[3];
    real fext[6];
    TrigC<real> trig;
};

// Forward-mode dual scalar: value v and tangent d = dv/dx for one seeded input x.  The recursions below are templated on
// their value type V (real, or Dual<real> for the derivative kernels); link constants stay real, so a product of a
// constant and a dual costs two multiplies, not the four of a dual-by-dual product.
template <typename real>
struct Dual {
    real v, d;
    Dual() = default;
    __device__ __forceinline__ Dual(real x) : v(x), d(0) {}
    __device__ __forceinline__ Dual(real x, real dx) : v(x), d(dx) {}
    __device__ __forceinline__ Dual operator-() const { return {-v, -d}; }
    __device__ __forceinline__ Dual &operator+=(Dual b) { v += b.v; d += b.d; return *this; }
    __device__ __forceinline__ Dual &operator+=(real b) { v += b; return *this; }
    friend __device__ __forceinline__ Dual operator+(Dual a, Dual b) { return {a.v + b.v, a.d + b.d}; }
    friend __device__ __forceinline__ Dual operator+(Dual a, real b) { return {a.v + b, a.d}; }
    friend __device__ __forceinline__ Dual operator+(real a, Dual b) { return {a + b.v, b.d}; }
    friend __device__ __forceinline__ Dual operator-(Dual a, Dual b) { return {a.v - b.v, a.d - b.d}; }
    friend __device__ __forceinline__ Dual operator*(Dual a, Dual b) { return {a.v * b.v, fma(a.v, b.d, a.d * b.v)}; }
    friend __device__ __forceinline__ Dual operator*(real a, Dual b) { return {a * b.v, a * b.d}; }
    friend __device__ __forceinline__ Dual operator*(Dual a, real b) { return {a.v * b, a.d * b}; }
    friend __device__ __forceinline__ Dual fma(Dual a, Dual b, Dual c) { return {fma(a.v, b.v, c.v), fma(a.v, b.d, fma(a.d, b.v, c.d))}; }
    friend __device__ __forceinline__ Dual fma(real a, Dual b, Dual c) { return {fma(a, b.v, c.v), fma(a, b.d, c.d)}; }
    friend __device__ __forceinline__ Dual fma(Dual a, real b, Dual c) { return {fma(a.v, b, c.v), fma(a.d, b, c.d)}; }
    friend __device__ __forceinline__ Dual fma(Dual a, Dual b, real c) { return {fma(a.v, b.v, c), fma(a.v, b.d, a.d * b.v)}; }
    friend __device__ __forceinline__ Dual fma(real a, Dual b, real c) { return {fma(a, b.v, c), a * b.d}; }
    friend __device__ __forceinline__ Dual fma(Dual a, real b, real c) { return {fma(a.v, b, c), a.d * b}; }
    friend __device__ __forceinline__ Dual fma(real a, real b, Dual c) { return {fma(a, b, c.v), c.d}; }
    // branches (Coulomb friction) follow the value: the tangent of a piecewise-constant term is 0
    friend __device__ __forceinline__ bool operator>(Dual a, real b) { return a.v > b; }
    friend __device__ __forceinline__ bool operator<(Dual a, real b) { return a.v < b; }
};

template <typename real>
struct V3 {
    real x, y, z;
};
// Mixed operands (a dual vector and a constant one) give a vector of the wider type; with one type they are the plain ops.
template <typename A, typename B>
__device__ __forceinline__ auto vadd(V3<A> a, V3<B> b) -> V3<decltype(a.x + b.x)> { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <typename A, typename B>
__device__ __forceinline__ auto vcross(V3<A> a, V3<B> b) -> V3<decltype(a.x * b.x)>
{
    return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
// a x b + c with the addition folded into the products (2 FMA per component instead of MUL + FMA + ADD)
template <typename A, typename B, typename C>
__device__ __forceinline__ V3<C> vcross_acc(V3<A> a, V3<B> b, V3<C> c)
{
    return {fma(a.y, b.z, fma(-a.z, b.y, c.x)), fma(a.z, b.x, fma(-a.x, b.z, c.y)), fma(a.x, b.y, fma(-a.y, b.x, c.z))};
}
template <typename V, typename real> __device__ __forceinline__ V3<V> vscale(V3<V> a, real s) { return {s * a.x, s * a.y, s * a.z}; }
template <typename A, typename B>
__device__ __forceinline__ auto vdot(V3<A> a, V3<B> b) -> decltype(a.x * b.x) { return a.x * b.x + a.y * b.y + a.z * b.z; }

// link rotation R (columns n, o, a) from sin/cos(theta), sin/cos(alpha); frne.c:329-347
template <typename real, bool MDH, typename V = real>
struct LinkRot {
    V nx, ny, nz, ox, oy, oz, ax, ay, az;
    __device__ __forceinline__ LinkRot(V st, V ct, real sa, real ca)
    {
        if (!MDH) {
            nx = ct; ox = -ca * st; ax = sa * st;
            ny = st; oy = ca * ct;  ay = -sa * ct;
            nz = 0;  oz = sa;       az = ca;
        } else {
            nx = ct;      ox = -st;     ax = 0;
            ny = st * ca; oy = ca * ct; ay = -sa;
            nz = st * sa; oz = ct * sa; az = ca;
        }
    }
    __device__ __forceinline__ V3<V> mul(V3<V> v) const
    {
        return {nx * v.x + ox * v.y + ax * v.z, ny * v.x + oy * v.y + ay * v.z, nz * v.x + oz * v.y + az * v.z};
    }
    __device__ __forceinline__ V3<V> tmul(V3<V> v) const
    {
        return {nx * v.x + ny * v.y + nz * v.z, ox * v.x + oy * v.y + oz * v.z, ax * v.x + ay * v.y + az * v.z};
    }
};

// ------------------------------------------------------------------ all-revolute fast path
// The same recursion as ne.c with the link rotation applied in its factored form
// (R = Rz(theta) Rx(alpha) for DH, Rx(alpha) Rz(theta) for MDH: 8 flops instead of the 9-entry
// product with its structural zeros), z-only joint-rate vectors expanded by hand (the compiler
// may not drop IEEE multiplications by a literal 0), p* taken from the constant bank, and
// R_{j+1} f_{j+1} computed once per link.  Dropping exact-zero terms does not change any value.
template <typename real, bool MDH, typename V = real>
struct FRot { // factored link rotation
    V st, ct;
    real sa, ca;
    template <typename X> __device__ __forceinline__ V3<V> tmul(V3<X> v) const // R^T v
    {
        if (!MDH) {
            const auto u = fma(ct, v.x, st * v.y), w = fma(ct, v.y, -(st * v.x));
            return {u, fma(ca, w, sa * v.z), fma(ca, v.z, -(sa * w))};
        } else {
            const auto wy = fma(ca, v.y, sa * v.z), wz = fma(ca, v.z, -(sa * v.y));
            return {fma(ct, v.x, st * wy), fma(ct, wy, -(st * v.x)), wz};
        }
    }
    template <typename X> __device__ __forceinline__ V3<V> mul(V3<X> v) const // R v
    {
        if (!MDH) {
            const auto m = fma(ca, v.y, -(sa * v.z)), z = fma(sa, v.y, ca * v.z);
            return {fma(ct, v.x, -(st * m)), fma(st, v.x, ct * m), z};
        } else {
            const auto u = fma(ct, v.x, -(st * v.y)), w = fma(st, v.x, ct * v.y);
            return {u, fma(ca, w, -(sa * v.z)), fma(sa, w, ca * v.z)};
        }
    }
    // R^T v + c and R v + c with c folded into the last stage of FMAs (no separate additions)
    __device__ __forceinline__ V3<V> tmul_acc(V3<V> v, V3<V> c) const
    {
        if (!MDH) {
            const auto w = fma(ct, v.y, -(st * v.x));
            return {fma(ct, v.x, fma(st, v.y, c.x)), fma(ca, w, fma(sa, v.z, c.y)), fma(ca, v.z, fma(-sa, w, c.z))};
        } else {
            const auto wy = fma(ca, v.y, sa * v.z);
            return {fma(ct, v.x, fma(st, wy, c.x)), fma(ct, wy, fma(-st, v.x, c.y)), fma(ca, v.z, fma(-sa, v.y, c.z))};
        }
    }
    __device__ __forceinline__ V3<V> mul_acc(V3<V> v, V3<V> c) const
    {
        if (!MDH) {
            const auto m = fma(ca, v.y, -(sa * v.z));
            return {fma(ct, v.x, fma(-st, m, c.x)), fma(st, v.x, fma(ct, m, c.y)), fma(sa, v.y, fma(ca, v.z, c.z))};
        } else {
            const auto w = fma(st, v.x, ct * v.y);
            return {fma(ct, v.x, fma(-st, v.y, c.x)), fma(ca, w, fma(-sa, v.z, c.y)), fma(sa, w, fma(ca, v.z, c.z))};
        }
    }
};

template <typename real, typename V>
__device__ __forceinline__ V3<V> imul(const real *I, V3<V> v) // vmath.c mat_vect_mult (column-major read)
{
    return {fma(I[0], v.x, fma(I[3], v.y, I[6] * v.z)), fma(I[1], v.x, fma(I[4], v.y, I[7] * v.z)),
            fma(I[2], v.x, fma(I[5], v.y, I[8] * v.z))};
}

// sin / cos of every link's joint angle as one interleaved batch (frne.c:193-207 rot_mat); prismatic
// links use the fixed theta of the link
template <typename real, int N, bool ALLREV>
__device__ __forceinline__ void rne_sincos(const RneP<real, N> &P, const real *mq, real *sth, real *cth)
{
    real th[N];
#pragma unroll
    for (int j = 0; j < N; j++) th[j] = mq[j] + P.offset[j];
    b2k_sincos_batch<real, N>(th, P.trig, sth, cth);
    if (!ALLREV) {
#pragma unroll
        for (int j = 0; j < N; j++)
            if (P.prismatic[j]) { sth[j] = P.st0[j]; cth[j] = P.ct0[j]; }
    }
}

// The base wrench (WRENCH): the force and moment the base exerts on link 1, in frame 0, the moment about the origin of
// frame 0: wb = [R_1 f_1, R_1 n_1] for DH (n_1 is already about O_0), [R_1 f_1, R_1 n_1 + p*_1 x R_1 f_1] for MDH
// (n_1 is about O_1: one more step of the backward recursion, onto a massless link 0).  The actuator terms act inside
// the joints and do not enter it.
template <typename real>
__device__ __forceinline__ void rne_put_wrench(V3<real> f0, V3<real> n0, real *wb)
{
    wb[0] = f0.x; wb[1] = f0.y; wb[2] = f0.z;
    wb[3] = n0.x; wb[4] = n0.y; wb[5] = n0.z;
}

template <typename real, int N, bool MDH, bool WRENCH = false, typename V = real>
__device__ __forceinline__ void rne_row_allrev(const RneP<real, N> &P, const V *sth, const V *cth, const V *mqd,
                                               const V *mqdd, V3<V> gravity, V *tq, V *wb = nullptr)
{
    V3<V> Fm[N], Nm[N];
    V3<V> w = {0, 0, 0}, wd = {0, 0, 0}, acc = {0, 0, 0};
#pragma unroll
    for (int j = 0; j < N; j++) {
        const FRot<real, MDH, V> R = {sth[j], cth[j], P.sa[j], P.ca[j]};
        const V3<real> ps = {P.ps[j][0], P.ps[j][1], P.ps[j][2]};
        const V qd = mqd[j], qdd = mqdd[j];
        V3<V> wn, wdn, accn;
        if (MDH) { // ne.c:144-181
            if (j == 0) {
                wn = {0, 0, qd};
                wdn = {0, 0, qdd};
                accn = R.tmul(gravity);
            } else {
                const V3<V> t1 = R.tmul(w);
                wn = {t1.x, t1.y, t1.z + qd};
                const V3<V> t3 = R.tmul(wd);
                wdn = {fma(t1.y, qd, t3.x), fma(-t1.x, qd, t3.y), t3.z + qdd}; // t1 x (0,0,qd) + t3 + (0,0,qdd)
                V3<V> a = vcross(w, ps);
                a = vcross_acc(w, a, acc);
                a = vcross_acc(wd, ps, a);
                accn = R.tmul(a);
            }
        } else { // ne.c:252-288
            if (j == 0) {
                wn = R.tmul(V3<V>{0, 0, qd});
                wdn = R.tmul(V3<V>{0, 0, qdd});
            } else {
                wn = R.tmul(V3<V>{w.x, w.y, w.z + qd});
                wdn = R.tmul(V3<V>{fma(w.y, qd, wd.x), fma(-w.x, qd, wd.y), wd.z + qdd});
            }
            const V3<V> t2 = vcross(wn, ps);
            accn = R.tmul_acc(j == 0 ? gravity : acc, vcross_acc(wdn, ps, vcross(wn, t2)));
        }
        w = wn; wd = wdn; acc = accn;
        const V3<real> rc = {P.r[j][0], P.r[j][1], P.r[j][2]};
        const V3<V> abar = vcross_acc(wd, rc, vcross_acc(w, vcross(w, rc), acc));
        Fm[j] = vscale(abar, P.m[j]);
        Nm[j] = vcross_acc(w, imul(P.I[j], w), imul(P.I[j], wd));
    }
    V3<V> f = {0, 0, 0}, nn = {0, 0, 0};
    const V3<real> f_tip = {P.fext[0], P.fext[1], P.fext[2]}, n_tip = {P.fext[3], P.fext[4], P.fext[5]};
#pragma unroll
    for (int j = N - 1; j >= 0; j--) {
        const V3<real> rc = {P.r[j][0], P.r[j][1], P.r[j][2]};
        V3<V> fj, nj;
        if (MDH) { // ne.c:358-398
            if (j == N - 1) {
                fj = vadd(f_tip, Fm[j]);
                nj = vadd(n_tip, Nm[j]);
            } else {
                const FRot<real, MDH, V> Rn = {sth[j + 1], cth[j + 1], P.sa[j + 1], P.ca[j + 1]};
                const V3<real> psn = {P.ps[j + 1][0], P.ps[j + 1][1], P.ps[j + 1][2]};
                const V3<V> Rf = Rn.mul(f);
                fj = vadd(Rf, Fm[j]);
                nj = Rn.mul_acc(nn, vcross_acc(psn, Rf, Nm[j]));
            }
            nj = vcross_acc(rc, Fm[j], nj);
        } else { // ne.c:409-453
            const V3<real> ps = {P.ps[j][0], P.ps[j][1], P.ps[j][2]};
            const V3<real> psrc = {P.psrc[j][0], P.psrc[j][1], P.psrc[j][2]};
            V3<V> t1 = vcross_acc(psrc, Fm[j], Nm[j]);
            if (j != N - 1) {
                const FRot<real, MDH, V> Rn = {sth[j + 1], cth[j + 1], P.sa[j + 1], P.ca[j + 1]};
                fj = Rn.mul_acc(f, Fm[j]);
                const V3<V> t3 = vcross_acc(Rn.tmul(ps), f, nn);
                t1 = Rn.mul_acc(t3, t1);
            } else {
                fj = vadd(Fm[j], f_tip);
                t1 = vadd(vcross_acc(ps, f_tip, t1), n_tip);
            }
            nj = t1;
        }
        f = fj; nn = nj;
        V t = MDH ? nj.z : fma(nj.y, P.sa[j], nj.z * P.ca[j]); // n . (R^T z0)
        const V qdj = mqd[j];
        t = fma(P.c_jm[j], mqdd[j], t);
        t = fma(P.c_b[j], qdj, t);
        t += (qdj > 0 ? P.c_tcp[j] : (real)0) + (qdj < 0 ? P.c_tcm[j] : (real)0);
        tq[j] = t;
    }
    if constexpr (WRENCH) {
        const FRot<real, MDH, V> R = {sth[0], cth[0], P.sa[0], P.ca[0]};
        const V3<V> f0 = R.mul(f);
        const V3<real> ps = {P.ps[0][0], P.ps[0][1], P.ps[0][2]};
        rne_put_wrench(f0, MDH ? R.mul_acc(nn, vcross(ps, f0)) : R.mul(nn), wb);
    }
}

// ------------------------------------------------------------------ generic row (any mix of revolute / prismatic links)
// Mirrors ne.c operation by operation, including its quirks for a prismatic first joint under
// modified DH (ne.c:187-204).
template <typename real, int N, bool MDH, bool WRENCH = false, typename V = real>
__device__ __forceinline__ void rne_row_generic(const RneP<real, N> &P, const V *mq, const V *sth, const V *cth,
                                                const V *mqd, const V *mqdd, V3<V> gravity, V *tq,
                                                V *wb = nullptr)
{
    // stash for the backward recursion
    V3<V> Fm[N], Nm[N];
    // (gravity: base acceleration handed in by the caller)
    V3<V> w = {0, 0, 0}, wd = {0, 0, 0}, acc = {0, 0, 0}; // of link j-1 on entry

    // ---------------- forward recursion (ne.c:137-240 MDH, 245-347 DH)
#pragma unroll
    for (int j = 0; j < N; j++) {
        const bool pris = (P.prismatic[j] != 0);
        const V st = sth[j], ct = cth[j];
        const V d = pris ? (mq[j] + P.offset[j]) : P.D[j];
        const LinkRot<real, MDH, V> R(st, ct, P.sa[j], P.ca[j]);
        const V3<V> pstar = MDH ? V3<V>{P.A[j], -d * P.sa[j], d * P.ca[j]} : V3<V>{P.A[j], d * P.sa[j], d * P.ca[j]};
        const V3<V> qdv = {0, 0, mqd[j]}, qddv = {0, 0, mqdd[j]};
        V3<V> wn, wdn, accn, t1, t2, t3;
        if (MDH) {
            if (!pris) {
                if (j == 0) {
                    wn = qdv; wdn = qddv; t1 = gravity;
                } else {
                    t1 = R.tmul(w);
                    wn = vadd(t1, qdv);
                    t3 = R.tmul(wd);
                    t2 = vcross(t1, qdv);
                    t1 = vadd(t2, t3);
                    wdn = vadd(t1, qddv);
                    t1 = vcross(w, pstar);
                    t2 = vcross(w, t1);
                    t1 = vcross(wd, pstar);
                    t1 = vadd(t1, t2);
                    t1 = vadd(t1, acc);
                }
                accn = R.tmul(t1);
            } else {
                if (j == 0) {
                    wn = qdv; wdn = qddv; accn = gravity; // sic, ne.c:187-204
                } else {
                    wn = R.tmul(w);
                    wdn = R.tmul(wd);
                    t1 = vcross(wd, pstar);
                    t3 = vcross(w, pstar);
                    t2 = vcross(w, t3);
                    t1 = vadd(t1, t2);
                    t1 = vadd(t1, acc);
                    accn = R.tmul(t1);
                    t2 = R.tmul(w);
                    t1 = vcross(t2, qdv);
                    t1 = vscale(t1, (real)2);
                    accn = vadd(accn, t1);
                    accn = vadd(accn, qddv);
                }
            }
        } else {
            if (!pris) {
                t1 = (j == 0) ? qdv : vadd(w, qdv);
                wn = R.tmul(t1);
                if (j == 0) t3 = qddv;
                else {
                    t1 = vadd(wd, qddv);
                    t2 = vcross(w, qdv);
                    t3 = vadd(t1, t2);
                }
                wdn = R.tmul(t3);
                t1 = vcross(wdn, pstar);
                t2 = vcross(wn, pstar);
                t3 = vcross(wn, t2);
                accn = vadd(t1, t3);
                t1 = R.tmul(j == 0 ? gravity : acc);
                accn = vadd(accn, t1);
            } else {
                if (j == 0) {
                    wn = {0, 0, 0}; wdn = {0, 0, 0};
                    t1 = vadd(qddv, gravity);
                    accn = R.tmul(t1);
                } else {
                    wn = R.tmul(w);
                    wdn = R.tmul(wd);
                    t1 = vadd(qddv, acc);
                    accn = R.tmul(t1);
                }
                t1 = vcross(wdn, pstar);
                accn = vadd(accn, t1);
                t1 = R.tmul(qdv);
                t2 = vcross(wn, t1);
                t2 = vscale(t2, (real)2);
                accn = vadd(accn, t2);
                t2 = vcross(wn, pstar);
                t3 = vcross(wn, t2);
                accn = vadd(accn, t3);
            }
        }
        w = wn; wd = wdn; acc = accn;
        // centre-of-mass acceleration, ne.c:228-232 / 335-339, then the link wrench terms
        const V3<real> rc = {P.r[j][0], P.r[j][1], P.r[j][2]};
        t1 = vcross(wd, rc);
        t2 = vcross(w, rc);
        t3 = vcross(w, t2);
        V3<V> abar = vadd(t1, t3);
        abar = vadd(abar, acc);
        Fm[j] = vscale(abar, P.m[j]);
        const real *I = P.I[j]; // read column-major like vmath.c mat_vect_mult
        t2 = {I[0] * wd.x + I[3] * wd.y + I[6] * wd.z, I[1] * wd.x + I[4] * wd.y + I[7] * wd.z,
              I[2] * wd.x + I[5] * wd.y + I[8] * wd.z};
        t3 = {I[0] * w.x + I[3] * w.y + I[6] * w.z, I[1] * w.x + I[4] * w.y + I[7] * w.z,
              I[2] * w.x + I[5] * w.y + I[8] * w.z};
        Nm[j] = vadd(t2, vcross(w, t3));
    }

    // ---------------- backward recursion (ne.c:358-403 MDH, 409-457 DH) + joint torque (ne.c:464-491)
    V3<V> f = {0, 0, 0}, nn = {0, 0, 0}; // of link j+1 on entry
    const V3<real> f_tip = {P.fext[0], P.fext[1], P.fext[2]}, n_tip = {P.fext[3], P.fext[4], P.fext[5]};
#pragma unroll
    for (int j = N - 1; j >= 0; j--) {
        const bool pris = (P.prismatic[j] != 0);
        const V3<real> rc = {P.r[j][0], P.r[j][1], P.r[j][2]};
        V3<V> fj, nj, t1, t2, t3, t4;
        if (MDH) {
            const V3<V> F = Fm[j];
            if (j == N - 1) {
                fj = vadd(f_tip, F);
                t1 = {n_tip.x, n_tip.y, n_tip.z};
            } else {
                const LinkRot<real, MDH, V> Rn(sth[j + 1], cth[j + 1], P.sa[j + 1], P.ca[j + 1]);
                const V dn = P.prismatic[j + 1] ? (mq[j + 1] + P.offset[j + 1]) : P.D[j + 1];
                const V3<V> pstar_n = {P.A[j + 1], -dn * P.sa[j + 1], dn * P.ca[j + 1]};
                t1 = Rn.mul(f);
                fj = vadd(t1, F);
                t1 = Rn.mul(nn);
                t4 = Rn.mul(f);
                t3 = vcross(pstar_n, t4);
                t1 = vadd(t1, t3);
            }
            t2 = vcross(rc, F);
            t1 = vadd(t1, t2);
            nj = vadd(t1, Nm[j]);
        } else {
            const V dj = pris ? (mq[j] + P.offset[j]) : P.D[j];
            const V3<V> pstar = {P.A[j], dj * P.sa[j], dj * P.ca[j]};
            t4 = Fm[j];
            t2 = vadd(pstar, rc);
            t1 = vcross(t2, t4);
            if (j != N - 1) {
                const LinkRot<real, MDH, V> Rn(sth[j + 1], cth[j + 1], P.sa[j + 1], P.ca[j + 1]);
                fj = vadd(t4, Rn.mul(f));
                t2 = Rn.tmul(pstar);
                t3 = vcross(t2, f);
                t3 = vadd(t3, nn);
                t2 = Rn.mul(t3);
                t1 = vadd(t1, t2);
            } else {
                fj = vadd(t4, f_tip);
                t2 = vcross(pstar, f_tip);
                t1 = vadd(t1, t2);
                t1 = vadd(t1, n_tip);
            }
            nj = vadd(t1, Nm[j]);
        }
        f = fj; nn = nj;
        // torque about / force along the joint axis
        V3<real> zax;
        if (MDH) zax = {0, 0, 1};
        else zax = {0, P.sa[j], P.ca[j]}; // R_j^T z0 = (n.z, o.z, a.z)
        V t = pris ? vdot(fj, zax) : vdot(nj, zax);
        const V qdj = mqd[j];
        t += P.c_jm[j] * mqdd[j];
        t += P.c_b[j] * qdj;
        t += (qdj > 0 ? P.c_tcp[j] : (real)0) + (qdj < 0 ? P.c_tcm[j] : (real)0);
        tq[j] = t;
    }
    if constexpr (WRENCH) { // the MDH prismatic-first-joint quirk above carries over: wb is what that recursion gives
        const LinkRot<real, MDH, V> R(sth[0], cth[0], P.sa[0], P.ca[0]);
        const V3<V> f0 = R.mul(f);
        V3<V> n0 = R.mul(nn);
        if (MDH) {
            const V d = P.prismatic[0] ? (mq[0] + P.offset[0]) : P.D[0];
            n0 = vadd(n0, vcross(V3<V>{P.A[0], -d * P.sa[0], d * P.ca[0]}, f0));
        }
        rne_put_wrench(f0, n0, wb);
    }
    // ---------------- stage tau and write it back coalesced

}

// ALLREV: every joint is revolute (the usual case) -- strips the prismatic code, which the compiler
// would otherwise if-convert into always-executed select chains.  WRENCH: also the base wrench of every row, staged
// behind tau in shared memory and written to its own (nrows, 6) array.
template <typename real, int N, bool MDH, bool ALLREV, bool WRENCH>
__device__ __forceinline__ void rne_tiles(const RneP<real, N> &P, const real *__restrict__ q, const real *__restrict__ qd,
                                          const real *__restrict__ qdd, long long nrows, real *__restrict__ tau,
                                          real *__restrict__ wbase_out, int warp_smem_bytes, int in_bytes, int qmode)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    unsigned char *wbase = smem_raw + (size_t)warp * warp_smem_bytes;
    real *sq = reinterpret_cast<real *>(wbase);
    real *sqd = reinterpret_cast<real *>(wbase + in_bytes);
    real *sqdd = reinterpret_cast<real *>(wbase + 2 * in_bytes);
    unsigned char *sout = wbase + 3 * in_bytes;
    const int lds = qmode ? N : (N | 1); // smem row stride of the input tiles
    const long long ntiles = (nrows + 31) >> 5;
    const long long tstride = (long long)gridDim.x * B2K_WARPS_PER_BLOCK;
    const float inv_n = 1.0f / (float)N;

    auto load_inputs = [&](long long t) {
        const long long r0 = t << 5;
        const int rh = (int)((nrows - r0) < 32 ? (nrows - r0) : 32);
        load_q_tile<real>(sq, q + r0 * N, rh, N, inv_n, qmode, lane);
        load_q_tile<real>(sqd, qd + r0 * N, rh, N, inv_n, qmode, lane);
        load_q_tile<real>(sqdd, qdd + r0 * N, rh, N, inv_n, qmode, lane);
    };
    long long tile = (long long)blockIdx.x * B2K_WARPS_PER_BLOCK + warp;
    if (tile < ntiles) load_inputs(tile);
    for (; tile < ntiles; tile += tstride) {
        const long long row0 = tile << 5;
        const int rows_here = (int)((nrows - row0) < 32 ? (nrows - row0) : 32);
        cp_async_wait_all();
        __syncwarp();
        const int myrow = (lane < rows_here ? lane : 0) * lds;
        const real *mq = sq + myrow, *mqd = sqd + myrow, *mqdd = sqdd + myrow;

        real tq[N], sth[N], cth[N], wb[6];
        rne_sincos<real, N, ALLREV>(P, mq, sth, cth);
        const V3<real> grav = {P.grav[0], P.grav[1], P.grav[2]};
        if constexpr (ALLREV) rne_row_allrev<real, N, MDH, WRENCH>(P, sth, cth, mqd, mqdd, grav, tq, wb);
        else rne_row_generic<real, N, MDH, WRENCH>(P, mq, sth, cth, mqd, mqdd, grav, tq, wb);
        // the inputs of this tile are dead (tq holds the results): prefetch the next tile behind the drain
        __syncwarp();
        if (tile + tstride < ntiles) load_inputs(tile + tstride);
        TileStage<real, N>::put_row(sout, lane, tq);
        if constexpr (WRENCH) TileStage<real, 6>::put_row(sout + TileStage<real, N>::BYTES, lane, wb);
        __syncwarp();
        TileStage<real, N>::drain(sout, tau + row0 * N, rows_here, lane);
        if constexpr (WRENCH) TileStage<real, 6>::drain(sout + TileStage<real, N>::BYTES, wbase_out + row0 * 6, rows_here, lane);
        __syncwarp();
    }
    cp_async_wait_all();
}

template <typename real, int N, bool MDH, bool ALLREV>
__global__ void __launch_bounds__(B2K_THREADS, (sizeof(real) == 4 || (ALLREV && N <= 6)) ? 4 : 3)
k_rne(const __grid_constant__ RneP<real, N> P, const real *__restrict__ q, const real *__restrict__ qd,
      const real *__restrict__ qdd, long long nrows, real *__restrict__ tau, int warp_smem_bytes, int in_bytes,
      int qmode)
{
    rne_tiles<real, N, MDH, ALLREV, false>(P, q, qd, qdd, nrows, tau, nullptr, warp_smem_bytes, in_bytes, qmode);
}

template <typename real, int N, bool MDH, bool ALLREV>
__global__ void __launch_bounds__(B2K_THREADS, (sizeof(real) == 4 || (ALLREV && N <= 6)) ? 4 : 3)
k_rne_wrench(const __grid_constant__ RneP<real, N> P, const real *__restrict__ q, const real *__restrict__ qd,
             const real *__restrict__ qdd, long long nrows, real *__restrict__ tau, real *__restrict__ wbase,
             int warp_smem_bytes, int in_bytes, int qmode)
{
    rne_tiles<real, N, MDH, ALLREV, true>(P, q, qd, qdd, nrows, tau, wbase, warp_smem_bytes, in_bytes, qmode);
}

// ------------------------------------------------------------------ dynamics fan-outs of the recursion (SURVEY 8f-1)
// The reference's DynamicsMixin builds everything from repeated rne calls in Python loops
// (Dynamics.py): inertia = n calls with unit accelerations (752-758), gravload = one call with
// qd = qdd = 0 (912-915), itorque = one call without gravity (1456-1459), coriolis = n + n(n-1)/2
// calls on a friction-free copy (825-857), accel = inertia + one call + an n x n solve (490-503).
// Here one lane does all the calls of its row with the link rotations (sincos) computed once;
// the loops over unit vectors are runtime loops (code size of ONE recursion), the small n x n
// accumulators live in local memory.
// MODE of k_rne_fan: the operation's offset from B2K_GEN_INERTIA
enum { FAN_INERTIA = 0, FAN_GRAVLOAD = 1, FAN_ITORQUE = 2, FAN_CORIOLIS = 3, FAN_ACCEL = 4 };
static_assert(B2K_GEN_INERTIA + FAN_GRAVLOAD == B2K_GEN_GRAVLOAD && B2K_GEN_INERTIA + FAN_ITORQUE == B2K_GEN_ITORQUE &&
                  B2K_GEN_INERTIA + FAN_CORIOLIS == B2K_GEN_CORIOLIS && B2K_GEN_INERTIA + FAN_ACCEL == B2K_GEN_ACCEL,
              "FAN_* = B2K_GEN_* - B2K_GEN_INERTIA");

template <int MODE, int N>
struct FanShape {
    static constexpr int NIN = B2K_RNE_OPS[B2K_GEN_INERTIA + MODE].nin;
    static constexpr int OUT = B2K_RNE_OPS[B2K_GEN_INERTIA + MODE].out_row(0, N);
};

// Solves A X = B by Gaussian elimination with partial pivoting (numpy.linalg.solve = LAPACK gesv), A = M (N x N,
// row-major, destroyed), B = rhs (N x NRHS, row-major, destroyed), X into x (N x NRHS)
template <typename real, int N, int NRHS>
__device__ __forceinline__ void rne_lu_solve(real *M, real *rhs, real *x)
{
#pragma unroll 1
    for (int c = 0; c < N; c++) {
        int p = c;
        real best = fabs(M[c * N + c]);
#pragma unroll 1
        for (int r = c + 1; r < N; r++) {
            const real v = fabs(M[r * N + c]);
            if (v > best) { best = v; p = r; }
        }
        if (p != c) {
#pragma unroll 1
            for (int k = 0; k < N; k++) { const real t = M[c * N + k]; M[c * N + k] = M[p * N + k]; M[p * N + k] = t; }
#pragma unroll
            for (int s = 0; s < NRHS; s++) { const real t = rhs[c * NRHS + s]; rhs[c * NRHS + s] = rhs[p * NRHS + s]; rhs[p * NRHS + s] = t; }
        }
        const real inv = (real)1 / M[c * N + c];
#pragma unroll 1
        for (int r = c + 1; r < N; r++) {
            const real f = M[r * N + c] * inv;
#pragma unroll 1
            for (int k = c; k < N; k++) M[r * N + k] -= f * M[c * N + k];
#pragma unroll
            for (int s = 0; s < NRHS; s++) rhs[r * NRHS + s] -= f * rhs[c * NRHS + s];
        }
    }
#pragma unroll 1
    for (int r = N - 1; r >= 0; r--) {
#pragma unroll
        for (int s = 0; s < NRHS; s++) {
            real acc = rhs[r * NRHS + s];
#pragma unroll 1
            for (int k = r + 1; k < N; k++) acc -= M[r * N + k] * x[k * NRHS + s];
            x[r * NRHS + s] = acc / M[r * N + r];
        }
    }
}

template <typename real, int N, bool MDH, bool ALLREV, int MODE>
__global__ void __launch_bounds__(B2K_THREADS, (sizeof(real) == 4) ? 3 : 2)
k_rne_fan(const __grid_constant__ RneP<real, N> P, const real *__restrict__ in0, const real *__restrict__ in1,
          const real *__restrict__ in2, long long nrows, real *__restrict__ out, int warp_smem_bytes, int in_bytes,
          int qmode)
{
    typedef FanShape<MODE, N> SH;
    typedef TileStage<real, SH::OUT> OS;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    unsigned char *wbase = smem_raw + (size_t)warp * warp_smem_bytes;
    real *s0 = reinterpret_cast<real *>(wbase);
    real *s1 = reinterpret_cast<real *>(wbase + in_bytes);
    real *s2 = reinterpret_cast<real *>(wbase + 2 * in_bytes);
    unsigned char *sout = wbase + SH::NIN * in_bytes;
    const int lds = qmode ? N : (N | 1);
    const long long ntiles = (nrows + 31) >> 5;
    const float inv_n = 1.0f / (float)N;
    const long long tile = (long long)blockIdx.x * B2K_WARPS_PER_BLOCK + warp; // one tile per warp, one-shot grid
    if (tile >= ntiles) return;
    const long long row0 = tile << 5;
    const int rows_here = (int)((nrows - row0) < 32 ? (nrows - row0) : 32);
    load_q_tile<real>(s0, in0 + row0 * N, rows_here, N, inv_n, qmode, lane);
    if (SH::NIN >= 2) load_q_tile<real>(s1, in1 + row0 * N, rows_here, N, inv_n, qmode, lane);
    if (SH::NIN >= 3) load_q_tile<real>(s2, in2 + row0 * N, rows_here, N, inv_n, qmode, lane);
    cp_async_wait_all();
    __syncwarp();
    const int myrow = (lane < rows_here ? lane : 0) * lds;
    const real *mq = s0 + myrow;

    real sth[N], cth[N];
    rne_sincos<real, N, ALLREV>(P, mq, sth, cth);
    const V3<real> gvec = {P.grav[0], P.grav[1], P.grav[2]}, gzero = {0, 0, 0};
    auto rne_eval_g = [&](const real *qdv, const real *qddv, V3<real> g, real *tq) {
        if constexpr (ALLREV) rne_row_allrev<real, N, MDH>(P, sth, cth, qdv, qddv, g, tq);
        else rne_row_generic<real, N, MDH>(P, mq, sth, cth, qdv, qddv, g, tq);
    };
    auto rne_eval = [&](const real *qdv, const real *qddv, real *tq) { rne_eval_g(qdv, qddv, gvec, tq); };
    real res[SH::OUT];
    real zero[N];
#pragma unroll
    for (int k = 0; k < N; k++) zero[k] = 0;

    if constexpr (MODE == FAN_GRAVLOAD) {
        rne_eval(zero, zero, res);
    } else if constexpr (MODE == FAN_ITORQUE) {
        real a[N];
#pragma unroll
        for (int k = 0; k < N; k++) a[k] = s1[myrow + k];
        rne_eval(zero, a, res);
    } else if constexpr (MODE == FAN_INERTIA) {
#pragma unroll 1
        for (int i = 0; i < N; i++) {
            real a[N], tq[N];
#pragma unroll
            for (int k = 0; k < N; k++) a[k] = (k == i) ? (real)1 : (real)0;
            rne_eval(zero, a, tq);
#pragma unroll
            for (int k = 0; k < N; k++) res[i * N + k] = tq[k]; // row i = torque for a unit acceleration of joint i
        }
    } else if constexpr (MODE == FAN_CORIOLIS) {
        real Csq[N * N];
        real qd[N];
#pragma unroll
        for (int k = 0; k < N; k++) qd[k] = s1[myrow + k];
#pragma unroll
        for (int k = 0; k < N * N; k++) res[k] = 0;
#pragma unroll 1
        for (int i = 0; i < N; i++) { // centripetal terms: one joint moving at unit speed (Dynamics.py:828-833)
            real v[N], tq[N];
#pragma unroll
            for (int k = 0; k < N; k++) v[k] = (k == i) ? (real)1 : (real)0;
            rne_eval(v, zero, tq);
#pragma unroll
            for (int k = 0; k < N; k++) Csq[k * N + i] = tq[k];
        }
#pragma unroll 1
        for (int i = 0; i < N; i++) { // Coriolis terms: pairs of joints at unit speed (Dynamics.py:839-855)
#pragma unroll 1
            for (int j = i + 1; j < N; j++) {
                real v[N], tq[N];
#pragma unroll
                for (int k = 0; k < N; k++) v[k] = (k == i || k == j) ? (real)1 : (real)0;
                rne_eval(v, zero, tq);
                real qdi = 0, qdj = 0;
#pragma unroll
                for (int k = 0; k < N; k++) { qdi = (k == i) ? qd[k] : qdi; qdj = (k == j) ? qd[k] : qdj; }
#pragma unroll
                for (int k = 0; k < N; k++) {
                    const real t = tq[k] - Csq[k * N + j] - Csq[k * N + i];
                    res[k * N + j] = res[k * N + j] + t * qdi / (real)2;
                    res[k * N + i] = res[k * N + i] + t * qdj / (real)2;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < N; k++)
#pragma unroll
            for (int i = 0; i < N; i++) res[k * N + i] = res[k * N + i] + Csq[k * N + i] * qd[i]; // + Csq @ diag(qd)
    } else { // FAN_ACCEL: qdd = M^-1 (tau - rne(q, qd, 0))  (Dynamics.py:490-503, Walker & Orin method 1)
        real M[N * N], rhs[N];
        {
            real v[N], tq[N];
#pragma unroll
            for (int k = 0; k < N; k++) v[k] = s1[myrow + k];
            rne_eval(v, zero, tq); // gravity + Coriolis + friction torque at zero acceleration
#pragma unroll
            for (int k = 0; k < N; k++) rhs[k] = s2[myrow + k] - tq[k];
        }
#pragma unroll 1
        for (int i = 0; i < N; i++) { // inertia rows: unit accelerations, no velocity, no gravity (Dynamics.py:492-496)
            real a[N], tq[N];
#pragma unroll
            for (int k = 0; k < N; k++) a[k] = (k == i) ? (real)1 : (real)0;
            rne_eval_g(zero, a, gzero, tq);
#pragma unroll
            for (int k = 0; k < N; k++) M[i * N + k] = tq[k];
        }
        rne_lu_solve<real, N, 1>(M, rhs, res);
    }
    OS::put_row(sout, lane, res);
    if (!OS::drain_async(sout, out + row0 * SH::OUT, rows_here, lane)) {
        __syncwarp();
        OS::drain(sout, out + row0 * SH::OUT, rows_here, lane);
    }
    OS::wait_all();
}

template <typename real, int N>
void rne_fill_params(const b2k_rne_s *r, const double *grav, const double *fext, RneP<real, N> &P)
{
    for (int j = 0; j < N; j++) {
        const double *l = r->L[j];
        const double alpha = l[0], A = l[1], theta = l[2], D = l[3], offset = l[5];
        const double G = l[20];
        P.sa[j] = (real)sin(alpha);
        P.ca[j] = (real)cos(alpha);
        P.A[j] = (real)A;
        P.D[j] = (real)D;
        P.st0[j] = (real)sin(theta);
        P.ct0[j] = (real)cos(theta);
        P.offset[j] = (real)offset;
        P.prismatic[j] = ((int)l[4]) != 0;
        P.m[j] = (real)l[6];
        for (int k = 0; k < 3; k++) P.r[j][k] = (real)l[7 + k];
        for (int k = 0; k < 9; k++) P.I[j][k] = (real)l[10 + k];
        P.c_jm[j] = (real)(G * G * l[19]);
        P.c_b[j] = (real)(G * G * l[21]);
        P.c_tcp[j] = (real)(fabs(G) * l[22]);
        P.c_tcm[j] = (real)(fabs(G) * l[23]);
        P.ps[j][0] = (real)A;
        P.ps[j][1] = (real)(r->mdh ? -D * sin(alpha) : D * sin(alpha));
        P.ps[j][2] = (real)(D * cos(alpha));
        for (int k = 0; k < 3; k++) P.psrc[j][k] = (real)((double)P.ps[j][k] + (double)P.r[j][k]);
    }
    for (int k = 0; k < 3; k++) P.grav[k] = grav ? (real)grav[k] : (real)0;
    for (int k = 0; k < 6; k++) P.fext[k] = fext ? (real)fext[k] : (real)0;
    b2k_fill_trig<real>(P.trig);
}

// ------------------------------------------------------------------ analytical derivatives of the recursion (DESIGN f-13)
// DERIV_INVERSE: in = (q, qd, qdd); out0 = dtau/dq, out1 = dtau/dqd (N, n, n), [i, k] = dtau_i / dx_k, tau exactly what
//                k_rne computes with the same gravity and tip wrench.
// DERIV_FORWARD: in = (q, qd, torque); with M = inertia(q) (the FAN_INERTIA layout) and qdd* = M^-1 (torque - rne(q, qd, 0))
//                as FAN_ACCEL computes them: out0 = -M^-1 dtau/dq, out1 = -M^-1 dtau/dqd (both at qdd*), out2 = M^-1.
// Column k of each Jacobian is one evaluation of the recursion on Dual<real>, seeded with the tangent of q_k (of
// sin / cos theta_k for a revolute joint, of d_k = q_k + offset_k for a prismatic one) or of qd_k.  Like the fan-outs,
// the loops over columns are runtime loops (code size of one dual recursion) and the n x n results live in local memory.
enum { DERIV_INVERSE = 0, DERIV_FORWARD = 1 };

template <typename real, int N, bool MDH, bool ALLREV, int MODE>
__global__ void __launch_bounds__(B2K_THREADS, (sizeof(real) == 4) ? 3 : 2)
k_rne_deriv(const __grid_constant__ RneP<real, N> P, const real *__restrict__ in0, const real *__restrict__ in1,
            const real *__restrict__ in2, long long nrows, real *__restrict__ out0, real *__restrict__ out1,
            real *__restrict__ out2, int warp_smem_bytes, int in_bytes, int qmode)
{
    typedef TileStage<real, N * N> OS;
    typedef Dual<real> D;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    unsigned char *wbase = smem_raw + (size_t)warp * warp_smem_bytes;
    real *s0 = reinterpret_cast<real *>(wbase);
    real *s1 = reinterpret_cast<real *>(wbase + in_bytes);
    real *s2 = reinterpret_cast<real *>(wbase + 2 * in_bytes);
    unsigned char *sout = wbase + 3 * in_bytes;
    const int lds = qmode ? N : (N | 1);
    const long long ntiles = (nrows + 31) >> 5;
    const float inv_n = 1.0f / (float)N;
    const long long tile = (long long)blockIdx.x * B2K_WARPS_PER_BLOCK + warp; // one tile per warp, one-shot grid
    if (tile >= ntiles) return;
    const long long row0 = tile << 5;
    const int rows_here = (int)((nrows - row0) < 32 ? (nrows - row0) : 32);
    load_q_tile<real>(s0, in0 + row0 * N, rows_here, N, inv_n, qmode, lane);
    load_q_tile<real>(s1, in1 + row0 * N, rows_here, N, inv_n, qmode, lane);
    load_q_tile<real>(s2, in2 + row0 * N, rows_here, N, inv_n, qmode, lane);
    cp_async_wait_all();
    __syncwarp();
    const int myrow = (lane < rows_here ? lane : 0) * lds;
    const real *mq = s0 + myrow;

    real sth[N], cth[N], qd[N], qdd[N];
    rne_sincos<real, N, ALLREV>(P, mq, sth, cth);
#pragma unroll
    for (int k = 0; k < N; k++) qd[k] = s1[myrow + k];
    const V3<real> gvec = {P.grav[0], P.grav[1], P.grav[2]};
    // one n x n output: staged, copied out, and the stage free again before the next one is put
    auto emit = [&](const real *res, real *out) {
        OS::put_row(sout, lane, res);
        if (!OS::drain_async(sout, out + row0 * (N * N), rows_here, lane)) {
            __syncwarp();
            OS::drain(sout, out + row0 * (N * N), rows_here, lane);
        }
        OS::wait_all();
        __syncwarp();
    };

    real Minv[MODE == DERIV_FORWARD ? N * N : 1];
    if constexpr (MODE == DERIV_FORWARD) { // qdd* and M^-1 from one pivoted solve of M [X0 | X] = [torque - rne(q, qd, 0) | I]
        real M[N * N], B[N * (N + 1)], X[N * (N + 1)], zero[N];
#pragma unroll
        for (int k = 0; k < N; k++) zero[k] = 0;
        {
            real tq[N];
            if constexpr (ALLREV) rne_row_allrev<real, N, MDH>(P, sth, cth, qd, zero, gvec, tq);
            else rne_row_generic<real, N, MDH>(P, mq, sth, cth, qd, zero, gvec, tq);
#pragma unroll
            for (int k = 0; k < N; k++) {
                B[k * (N + 1)] = s2[myrow + k] - tq[k];
#pragma unroll
                for (int i = 0; i < N; i++) B[k * (N + 1) + 1 + i] = (k == i) ? (real)1 : (real)0;
            }
        }
#pragma unroll 1
        for (int i = 0; i < N; i++) { // inertia rows: unit accelerations, no velocity, no gravity (as FAN_ACCEL)
            real a[N], tq[N];
#pragma unroll
            for (int k = 0; k < N; k++) a[k] = (k == i) ? (real)1 : (real)0;
            if constexpr (ALLREV) rne_row_allrev<real, N, MDH>(P, sth, cth, zero, a, V3<real>{0, 0, 0}, tq);
            else rne_row_generic<real, N, MDH>(P, mq, sth, cth, zero, a, V3<real>{0, 0, 0}, tq);
#pragma unroll
            for (int k = 0; k < N; k++) M[i * N + k] = tq[k];
        }
        rne_lu_solve<real, N, N + 1>(M, B, X);
#pragma unroll
        for (int k = 0; k < N; k++) {
            qdd[k] = X[k * (N + 1)];
#pragma unroll
            for (int i = 0; i < N; i++) Minv[k * N + i] = X[k * (N + 1) + 1 + i];
        }
        emit(Minv, out2);
    } else {
#pragma unroll
        for (int k = 0; k < N; k++) qdd[k] = s2[myrow + k];
    }

    const V3<D> gdual = {gvec.x, gvec.y, gvec.z};
#pragma unroll 1
    for (int pass = 0; pass < 2; pass++) { // 0: columns of q, 1: columns of qd
        real res[N * N];
#pragma unroll 1
        for (int k = 0; k < N; k++) {
            D S[N], Cs[N], Q[N], QD[N], QDD[N], tq[N];
#pragma unroll
            for (int j = 0; j < N; j++) {
                const bool sq = pass == 0 && j == k;
                const bool rev = ALLREV || !P.prismatic[j];
                S[j] = D(sth[j], (sq && rev) ? cth[j] : (real)0);
                Cs[j] = D(cth[j], (sq && rev) ? -sth[j] : (real)0);
                Q[j] = D(mq[j], (sq && !rev) ? (real)1 : (real)0);
                QD[j] = D(qd[j], (pass == 1 && j == k) ? (real)1 : (real)0);
                QDD[j] = D(qdd[j]);
            }
            if constexpr (ALLREV) rne_row_allrev<real, N, MDH, false, D>(P, S, Cs, QD, QDD, gdual, tq);
            else rne_row_generic<real, N, MDH, false, D>(P, Q, S, Cs, QD, QDD, gdual, tq);
            if constexpr (MODE == DERIV_FORWARD) {
#pragma unroll
                for (int i = 0; i < N; i++) {
                    real acc = 0;
#pragma unroll
                    for (int j = 0; j < N; j++) acc = fma(Minv[i * N + j], tq[j].d, acc);
                    res[i * N + k] = -acc;
                }
            } else {
#pragma unroll
                for (int i = 0; i < N; i++) res[i * N + k] = tq[i].d;
            }
        }
        emit(res, pass == 0 ? out0 : out1);
    }
}

// ------------------------------------------------------------------ the dynamics regressor (DESIGN f-16)
// tau = Y(q, qd, qdd; g) pi without a tip wrench, pi = 14 parameters per link, link-major:
//   [m, m rx, m ry, m rz, Ixx, Iyy, Izz, Ixy, Iyz, Ixz, Jm, B, Tc+, Tc-]
// r the link's centre of mass in its frame, the inertia about the link-frame origin, I + m (r.r E - r r^T).
// Row j of Y is built from the unit twist s = (sf, sn) of joint j carried out along the chain: joint j's torque from a
// wrench (f, n) of link i >= j about O_i, in frame i, is sf . f + sn . n -- the transpose of the backward recursion of
// rne_row_generic, which carries the wrench of link i in to joint j.  The wrench of link i is linear in its parameters:
//   f = m a + wd x (m r) + w x (w x (m r)),   n = I_o wd + w x (I_o w) + (m r) x a
// with w, wd, a the angular velocity, angular acceleration and frame-origin acceleration (gravity included) of link i in
// its own frame, from the forward recursion below.

// One step of the forward recursion: link j's w, wd and acc from link j-1's.  The forward half of rne_row_generic,
// restated formula by formula with its quirks (ne.c:137-240 MDH, 245-347 DH; the MDH prismatic first joint, ne.c:187-204).
template <typename real, int N, bool MDH, bool ALLREV>
__device__ __forceinline__ void rne_forward_step(const RneP<real, N> &P, int j, const real *mq, const real *sth, const real *cth,
                                                 const real *mqd, const real *mqdd, V3<real> gravity, V3<real> &w, V3<real> &wd,
                                                 V3<real> &acc)
{
    typedef V3<real> V;
    const bool pris = !ALLREV && (P.prismatic[j] != 0);
    const real st = sth[j], ct = cth[j];
    const real d = pris ? (mq[j] + P.offset[j]) : P.D[j];
    const LinkRot<real, MDH> R(st, ct, P.sa[j], P.ca[j]);
    const V pstar = MDH ? V{P.A[j], -d * P.sa[j], d * P.ca[j]} : V{P.A[j], d * P.sa[j], d * P.ca[j]};
    const V qdv = {0, 0, mqd[j]}, qddv = {0, 0, mqdd[j]};
    V wn, wdn, accn, t1, t2, t3;
    if (MDH) {
        if (!pris) {
            if (j == 0) {
                wn = qdv; wdn = qddv; t1 = gravity;
            } else {
                t1 = R.tmul(w);
                wn = vadd(t1, qdv);
                t3 = R.tmul(wd);
                t2 = vcross(t1, qdv);
                t1 = vadd(t2, t3);
                wdn = vadd(t1, qddv);
                t1 = vcross(w, pstar);
                t2 = vcross(w, t1);
                t1 = vcross(wd, pstar);
                t1 = vadd(t1, t2);
                t1 = vadd(t1, acc);
            }
            accn = R.tmul(t1);
        } else {
            if (j == 0) {
                wn = qdv; wdn = qddv; accn = gravity; // sic, ne.c:187-204
            } else {
                wn = R.tmul(w);
                wdn = R.tmul(wd);
                t1 = vcross(wd, pstar);
                t3 = vcross(w, pstar);
                t2 = vcross(w, t3);
                t1 = vadd(t1, t2);
                t1 = vadd(t1, acc);
                accn = R.tmul(t1);
                t2 = R.tmul(w);
                t1 = vcross(t2, qdv);
                t1 = vscale(t1, (real)2);
                accn = vadd(accn, t1);
                accn = vadd(accn, qddv);
            }
        }
    } else {
        if (!pris) {
            t1 = (j == 0) ? qdv : vadd(w, qdv);
            wn = R.tmul(t1);
            if (j == 0) t3 = qddv;
            else {
                t1 = vadd(wd, qddv);
                t2 = vcross(w, qdv);
                t3 = vadd(t1, t2);
            }
            wdn = R.tmul(t3);
            t1 = vcross(wdn, pstar);
            t2 = vcross(wn, pstar);
            t3 = vcross(wn, t2);
            accn = vadd(t1, t3);
            t1 = R.tmul(j == 0 ? gravity : acc);
            accn = vadd(accn, t1);
        } else {
            if (j == 0) {
                wn = {0, 0, 0}; wdn = {0, 0, 0};
                t1 = vadd(qddv, gravity);
                accn = R.tmul(t1);
            } else {
                wn = R.tmul(w);
                wdn = R.tmul(wd);
                t1 = vadd(qddv, acc);
                accn = R.tmul(t1);
            }
            t1 = vcross(wdn, pstar);
            accn = vadd(accn, t1);
            t1 = R.tmul(qdv);
            t2 = vcross(wn, t1);
            t2 = vscale(t2, (real)2);
            accn = vadd(accn, t2);
            t2 = vcross(wn, pstar);
            t3 = vcross(wn, t2);
            accn = vadd(accn, t3);
        }
    }
    w = wn; wd = wdn; acc = accn;
}

// The per-warp slab of one joint row, and how it leaves so that every 32-byte sector of Y is written whole by one warp
// instruction.  A row of the batch is 14 N^2 reals, joint row j of it 14 N: these pieces start on a sector boundary only
// for some N and dtypes, so a sector can hold the end of joint row j and the start of j + 1, or the end of a row's last
// joint row and the start of the next row's first.  Slab row l (the tile's row l) is laid out from the sector boundary at
// or below the start of its joint row: [tail of joint row j - 1 | joint row j | start of the next row's joint row 0 (last
// j only)].  Joint row j leaves from its first sector boundary up to its last one; the partial sector at its end goes out
// with joint row j + 1 (the tail is carried to the front of the slab row), and the partial sector at the start of a row's
// joint row 0 waits in STASH until the previous row's last joint row, which completes the sector.  The warp drains one
// tile row at a time, consecutive lanes on consecutive reals from a sector boundary.  Where every joint row starts on a
// sector boundary the carry and the stash are empty and the tile drains as one sequence, all lanes busy.
template <typename real, int N>
struct RegSlab {
    static constexpr int ROW = 14 * N;
    static constexpr int SE = 32 / (int)sizeof(real); // reals per sector
    static constexpr int LD = (ROW + 2 * SE) | 1;     // slab row stride in reals
    static constexpr int STASH = 32 * LD;             // offset of the per-row stash of SE reals
    static constexpr int BYTES = ((32 * LD + 32 * SE) * (int)sizeof(real) + 15) & ~15;
};

template <typename real, int N, bool MDH, bool ALLREV>
__global__ void __launch_bounds__(B2K_THREADS, 1)
k_rne_regressor(const __grid_constant__ RneP<real, N> P, const real *__restrict__ in0, const real *__restrict__ in1,
                const real *__restrict__ in2, long long nrows, real *__restrict__ out, int warp_smem_bytes, int in_bytes,
                int qmode)
{
    typedef RegSlab<real, N> SL;
    typedef V3<real> V;
    constexpr int ROWN = 14 * N * N; // reals per row of the batch
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    unsigned char *wbase = smem_raw + (size_t)warp * warp_smem_bytes;
    real *s0 = reinterpret_cast<real *>(wbase);
    real *s1 = reinterpret_cast<real *>(wbase + in_bytes);
    real *s2 = reinterpret_cast<real *>(wbase + 2 * in_bytes);
    real *slab = reinterpret_cast<real *>(wbase + 3 * in_bytes);
    const int lds = qmode ? N : (N | 1);
    const long long ntiles = (nrows + 31) >> 5;
    const float inv_n = 1.0f / (float)N;
    const long long tile = (long long)blockIdx.x * B2K_WARPS_PER_BLOCK + warp; // one tile per warp, one-shot grid
    if (tile >= ntiles) return;
    const long long row0 = tile << 5;
    const int rows_here = (int)((nrows - row0) < 32 ? (nrows - row0) : 32);
    load_q_tile<real>(s0, in0 + row0 * N, rows_here, N, inv_n, qmode, lane);
    load_q_tile<real>(s1, in1 + row0 * N, rows_here, N, inv_n, qmode, lane);
    load_q_tile<real>(s2, in2 + row0 * N, rows_here, N, inv_n, qmode, lane);
    cp_async_wait_all();
    __syncwarp();
    const int myrow = (lane < rows_here ? lane : 0) * lds;
    const real *mq = s0 + myrow, *mqd = s1 + myrow, *mqdd = s2 + myrow;

    real sth[N], cth[N];
    rne_sincos<real, N, ALLREV>(P, mq, sth, cth);
    const V grav = {P.grav[0], P.grav[1], P.grav[2]};
    real *my = slab + lane * SL::LD;
    real *gtile = out + row0 * ROWN;
    constexpr int SE = SL::SE;
    // reals between joint row jr of tile row r and the sector boundary at or below it
    auto mis_of = [&](int r, int jr) { return (int)((reinterpret_cast<uintptr_t>(gtile + (long long)r * ROWN + jr * SL::ROW) & 31) / sizeof(real)); };
    int mis_prev = 0;
    // every joint row of every row starts on a sector boundary (fp64 with even N, fp32 with N divisible by 4, and Y
    // 32-byte aligned): no carry or stash is needed, and the tile drains as one sequence
    const bool whole = (SL::ROW * (int)sizeof(real)) % 32 == 0 && mis_of(0, 0) == 0;

#pragma unroll 1
    for (int jr = 0; jr < N; jr++) { // joint row jr of every row of the tile
        const int mis = mis_of(lane, jr);
        if (jr > 0) // the tail of joint row jr - 1 that did not fill its last sector
            for (int t = 0; t < mis; t++) my[t] = my[mis_prev + SL::ROW - mis + t];
        mis_prev = mis;
        V w = {0, 0, 0}, wd = {0, 0, 0}, acc = {0, 0, 0};
        V sf = {0, 0, 0}, sn = {0, 0, 0};
#pragma unroll
        for (int i = 0; i < N; i++) {
            rne_forward_step<real, N, MDH, ALLREV>(P, i, mq, sth, cth, mqd, mqdd, grav, w, wd, acc);
            real *y = my + mis + 14 * i;
            if (i < jr) {
#pragma unroll
                for (int k = 0; k < 14; k++) y[k] = 0;
                continue;
            }
            const bool pris = !ALLREV && (P.prismatic[i] != 0);
            const real d = pris ? (mq[i] + P.offset[i]) : P.D[i];
            const V ps = MDH ? V{P.A[i], -d * P.sa[i], d * P.ca[i]} : V{P.A[i], d * P.sa[i], d * P.ca[i]};
            if (i == jr) { // joint jr's own unit twist, as rne_row_generic projects its wrench
                const V z = MDH ? V{0, 0, 1} : V{0, P.sa[i], P.ca[i]}; // MDH: z of frame i; DH: R_i^T z0 (axis on frame i-1)
                if (pris) { sf = z; sn = {0, 0, 0}; }
                else { sn = z; sf = MDH ? V{0, 0, 0} : vcross(z, ps); } // DH: the moment is taken about O_{i-1} = O_i - p*
            } else { // carried out through joint i: the transpose of the backward step
                const LinkRot<real, MDH> R(sth[i], cth[i], P.sa[i], P.ca[i]);
                if (MDH) {
                    sf = R.tmul(vadd(sf, vcross(sn, ps)));
                    sn = R.tmul(sn);
                } else {
                    sn = R.tmul(sn);
                    sf = vadd(R.tmul(sf), vcross(sn, ps));
                }
            }
            // the 10 inertial columns: the coefficients of m, m r and I_o in sf . f + sn . n
            y[0] = vdot(sf, acc);
            const V h = vadd(vadd(vcross(sf, wd), vscale(w, vdot(sf, w))), vadd(vscale(sf, -vdot(w, w)), vcross(acc, sn)));
            y[1] = h.x; y[2] = h.y; y[3] = h.z;
            const V u = vcross(sn, w); // sn . (w x I w) = u . I w
            y[4] = sn.x * wd.x + u.x * w.x;
            y[5] = sn.y * wd.y + u.y * w.y;
            y[6] = sn.z * wd.z + u.z * w.z;
            y[7] = sn.x * wd.y + sn.y * wd.x + u.x * w.y + u.y * w.x;
            y[8] = sn.y * wd.z + sn.z * wd.y + u.y * w.z + u.z * w.y;
            y[9] = sn.x * wd.z + sn.z * wd.x + u.x * w.z + u.z * w.x;
            // joint friction acts in joint i only; P holds the constants of a unit table: G^2, G^2, |G|, |G|
            const real qdi = mqd[i];
            const bool own = i == jr;
            y[10] = own ? P.c_jm[i] * mqdd[i] : (real)0;
            y[11] = own ? P.c_b[i] * qdi : (real)0;
            y[12] = own && qdi > 0 ? P.c_tcp[i] : (real)0;
            y[13] = own && qdi < 0 ? P.c_tcm[i] : (real)0;
        }
        if (jr == 0) // the start of joint row 0 up to its first sector boundary: written with the previous row's end
            for (int t = 0; t < (SE - mis) % SE; t++) slab[SL::STASH + lane * SE + t] = my[mis + t];
        const int end = mis + SL::ROW; // slab position of the end of joint row jr
        if (jr == N - 1) {
            __syncwarp();
            if (lane < rows_here - 1) // complete the last sector with the next row's stashed start
                for (int t = 0; t < (SE - end % SE) % SE; t++) my[end + t] = slab[SL::STASH + (lane + 1) * SE + t];
        }
        __syncwarp();
        if (whole) { // every piece starts on a sector boundary: the tile's pieces back to back, all lanes busy
            const int cnt = rows_here * SL::ROW;
            real *g = gtile + jr * SL::ROW;
            for (int e = lane; e < cnt; e += 32) {
                const int r = e / SL::ROW, c = e - r * SL::ROW;
                g[(long long)r * ROWN + c] = slab[r * SL::LD + c];
            }
        } else { // one tile row at a time from its first sector boundary, consecutive lanes on consecutive reals
            for (int r = 0; r < rows_here; r++) {
                const int m = mis_of(r, jr);
                const int e = m + SL::ROW;
                const int lo = jr > 0 ? 0 : (r > 0 ? m + (SE - m) % SE : m);
                const int hi = jr < N - 1 ? e - e % SE : (r < rows_here - 1 ? e + (SE - e % SE) % SE : e);
                real *g = gtile + (long long)r * ROWN + jr * SL::ROW - m; // the sector boundary at or below joint row jr
                for (int u = lo + lane; u < hi; u += 32) g[u] = slab[r * SL::LD + u];
            }
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------ normal equations of the regressor (DESIGN f-16)
// G = sum Y^T W Y, b = sum Y^T W tau, s = sum tau^T W tau over a batch, in fp64, without Y ever existing in full: the
// regressor kernel writes a chunk of REG_CHUNK rows into a stream-ordered scratch buffer, k_regressor_syrk folds it into
// per-(tile pair, slice) partials, k_regressor_gram_reduce sums the partials.  The three are one Gram matrix of the
// augmented rows [Y[row, j, :] | tau[row, j]] weighted by w_j.  Every sum runs in a fixed order: no atomics, two equal
// calls give equal bits.
constexpr long long REG_CHUNK = 4096; // rows per chunk: Puma560 fp64 is 16.5 MB of Y, well inside H100's 50 MB L2
constexpr int REG_TILE = 32;          // the Gram matrix in 32 x 32 tiles, upper triangle only
constexpr int REG_KB = 16;            // augmented rows per k-step

constexpr int REG_MAX_ROWS = 16; // joints (DH, up to B2K_MAX_JOINTS) or joint groups (trees, up to 16) per row of the batch

struct RegWeights {
    double w[REG_MAX_ROWS]; // W.w[k % n]: one weight per joint row
};

// tile pair t (row-major over the upper triangle of an nt x nt tiling) -> (ti, tj), ti <= tj
__device__ __forceinline__ void reg_tile_pair(int t, int nt, int &ti, int &tj)
{
    ti = 0;
    while (t >= nt - ti) { t -= nt - ti; ti++; }
    tj = ti + t;
}

// Block (tile pair, slice): 4 groups of 64 threads, each thread a 4 x 4 register tile of the 32 x 32 tile; group g takes
// every 4th k-step of the slice, and the groups are summed in order at the end.
template <typename real>
__global__ void __launch_bounds__(256)
k_regressor_syrk(const real *__restrict__ Y, const real *__restrict__ tau, long long K, int n, int p, int nt,
                 const __grid_constant__ RegWeights W,
                 double *__restrict__ part, int accumulate)
{
    __shared__ __align__(16) double sm[4][2][REG_KB][REG_TILE]; // per group: the A and B k-step tiles; then the group sums
    const int tid = threadIdx.x, g = tid >> 6, t = tid & 63, tx = t & 7, ty = t >> 3;
    int ti, tj;
    reg_tile_pair(blockIdx.x, nt, ti, tj);
    const long long nkb = (K + REG_KB - 1) / REG_KB;
    const long long b0 = nkb * blockIdx.y / gridDim.y, b1 = nkb * (blockIdx.y + 1) / gridDim.y;
    const long long rounds = (b1 - b0 + 3) / 4;
    double acc[4][4];
#pragma unroll
    for (int u = 0; u < 4; u++)
#pragma unroll
        for (int v = 0; v < 4; v++) acc[u][v] = 0;
    // K <= REG_CHUNK * n: 32-bit row arithmetic
    const int ca = ti * REG_TILE, cb = tj * REG_TILE;
    auto elem = [&](int k, int col) -> double {
        if (col > p) return 0.0;
        return col < p ? (double)Y[(size_t)k * p + col] : (double)tau[k];
    };
    for (long long rd = 0; rd < rounds; rd++) {
        const int kb = (int)(b0 + 4 * rd + g);
#pragma unroll
        for (int m = 0; m < REG_KB * REG_TILE / 64; m++) {
            const int e = t + 64 * m, kk = e / REG_TILE, cc = e % REG_TILE;
            const int k = kb * REG_KB + kk;
            const bool live = kb < b1 && k < K;
            sm[g][0][kk][cc] = live ? W.w[k % n] * elem(k, ca + cc) : 0.0;
            sm[g][1][kk][cc] = live ? elem(k, cb + cc) : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < REG_KB; kk++) {
            const double2 a01 = *reinterpret_cast<const double2 *>(&sm[g][0][kk][ty * 4]);
            const double2 a23 = *reinterpret_cast<const double2 *>(&sm[g][0][kk][ty * 4 + 2]);
            const double2 c01 = *reinterpret_cast<const double2 *>(&sm[g][1][kk][tx * 4]);
            const double2 c23 = *reinterpret_cast<const double2 *>(&sm[g][1][kk][tx * 4 + 2]);
            const double a[4] = {a01.x, a01.y, a23.x, a23.y}, c[4] = {c01.x, c01.y, c23.x, c23.y};
#pragma unroll
            for (int u = 0; u < 4; u++)
#pragma unroll
                for (int v = 0; v < 4; v++) acc[u][v] = fma(a[u], c[v], acc[u][v]);
        }
        __syncthreads();
    }
    double *red = &sm[0][0][0][0]; // 4 groups x 1024 sums
#pragma unroll
    for (int u = 0; u < 4; u++)
#pragma unroll
        for (int v = 0; v < 4; v++) red[g * 1024 + (ty * 4 + u) * REG_TILE + tx * 4 + v] = acc[u][v];
    __syncthreads();
    double *dst = part + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * (REG_TILE * REG_TILE);
#pragma unroll
    for (int m = 0; m < 4; m++) {
        const int e = tid + 256 * m;
        const double sum = ((red[e] + red[1024 + e]) + red[2048 + e]) + red[3072 + e];
        dst[e] = accumulate ? dst[e] + sum : sum;
    }
}

// entry (a, c) of the augmented (p + 1) x (p + 1) Gram matrix: the slices summed in order; (a, c) and (c, a) read the same
// partials in the same order, so G comes out exactly symmetric
template <int TILE>
__global__ void __launch_bounds__(256)
k_regressor_gram_reduce(const double *__restrict__ part, int slices, int npairs, int nt, int p, double *__restrict__ G,
                        double *__restrict__ b, double *__restrict__ s)
{
    const int P = p + 1;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P * P) return;
    const int a = idx / P, c = idx - a * P;
    const int lo = a < c ? a : c, hi = a < c ? c : a;
    const int ti = lo / TILE, tj = hi / TILE;
    const int t = ti * nt - ti * (ti - 1) / 2 + (tj - ti);
    const int e = (lo % TILE) * TILE + hi % TILE;
    double sum = 0;
    for (int sl = 0; sl < slices; sl++) sum += part[((size_t)sl * npairs + t) * (TILE * TILE) + e];
    if (a < p && c < p) G[(size_t)a * p + c] = sum;
    else if (a < p) b[a] = sum;
    else if (c == p) *s = sum;
}

// ------------------------------------------------------------------ the generic launch path of every operation
// The generic kernel of operation OP (B2K_GEN_*) for one link-table shape
template <typename real, int N, bool MDH, bool ALLREV, int OP>
constexpr auto rne_generic_kernel()
{
    if constexpr (OP == B2K_GEN_RNE) return k_rne<real, N, MDH, ALLREV>;
    else if constexpr (OP == B2K_GEN_RNE_WRENCH) return k_rne_wrench<real, N, MDH, ALLREV>;
    else if constexpr (OP == B2K_GEN_RNE_DERIV) return k_rne_deriv<real, N, MDH, ALLREV, DERIV_INVERSE>;
    else if constexpr (OP == B2K_GEN_ACCEL_DERIV) return k_rne_deriv<real, N, MDH, ALLREV, DERIV_FORWARD>;
    else if constexpr (OP == B2K_GEN_RNE_REGRESSOR) return k_rne_regressor<real, N, MDH, ALLREV>;
    else return k_rne_fan<real, N, MDH, ALLREV, OP - B2K_GEN_INERTIA>;
}

// One launch of operation OP's generic kernel over a.nrows rows: a one-shot grid, one 32-row tile per warp.  The caller
// (b2k_api.cu) has checked every array against B2K_RNE_OPS[OP], the outputs against their stage unit.
template <typename real, int N, int OP>
int rne_generic_launch_op(const b2k_rne_s *r, const b2k_rne_args &a, cudaStream_t st)
{
    constexpr b2k_rne_op_s op = B2K_RNE_OPS[OP];
    RneP<real, N> P;
    if constexpr (OP == B2K_GEN_RNE_REGRESSOR) { // the friction constants of a unit table: G^2, G^2, |G|, |G|
        b2k_rne_s unit = *r;
        for (int j = 0; j < N; j++) unit.L[j][19] = unit.L[j][21] = unit.L[j][22] = unit.L[j][23] = 1.0;
        rne_fill_params<real, N>(&unit, a.grav, nullptr, P);
    } else {
        rne_fill_params<real, N>(r, op.grav ? a.grav : nullptr, op.fext ? a.fext : nullptr, P);
    }
    if (OP == B2K_GEN_CORIOLIS) { // the reference works on robot.nofriction(True, True) (Dynamics.py:818)
        for (int j = 0; j < N; j++) { P.c_b[j] = 0; P.c_tcp[j] = 0; P.c_tcm[j] = 0; }
    }
    // per warp: the input tiles, then the output stage (the base wrench has its own behind tau's; the derivative
    // outputs take turns in one; the regressor's is the slab of one joint row)
    const size_t inb = fkj_q_bytes<real>(N);
    size_t stage;
    if constexpr (OP == B2K_GEN_RNE_REGRESSOR) stage = RegSlab<real, N>::BYTES;
    else stage = (size_t)TileStage<real, op.out_row(0, N)>::BYTES + (op.wrench ? (size_t)TileStage<real, 6>::BYTES : 0);
    const size_t wsm = (op.nin * inb + stage + 15) & ~(size_t)15;
    const size_t smem = wsm * B2K_WARPS_PER_BLOCK;
    const real *in[3] = {(const real *)a.in[0], (const real *)a.in[1], (const real *)a.in[2]};
    real *out[3] = {(real *)a.out[0], (real *)a.out[1], (real *)a.out[2]};
    int qmode = 1;
    for (int i = 0; i < op.nin; i++) qmode = qmode && fkj_qmode<real>(in[i], N);
    const long long ntiles = (a.nrows + 31) / 32;
    const unsigned grid = (unsigned)((ntiles + B2K_WARPS_PER_BLOCK - 1) / B2K_WARPS_PER_BLOCK);
    const char *what = OP == B2K_GEN_RNE || OP == B2K_GEN_RNE_WRENCH ? "rne"
                       : OP == B2K_GEN_RNE_REGRESSOR                 ? "rne regressor"
                       : OP >= B2K_GEN_RNE_DERIV                     ? "rne derivative"
                                                                     : "rne fan-out";
    auto launch = [&](auto kern) -> int {
        const int per_sm = b2k_blocks_per_sm((const void *)kern, B2K_THREADS, smem);
        if (per_sm < 1) return per_sm < 0 ? per_sm : (b2k_set_error("%s kernel does not fit on an SM", what), B2K_ERR_INVALID);
        if constexpr (B2K_RNE_OPS[OP].nout == 1) kern<<<grid, B2K_THREADS, smem, st>>>(P, in[0], in[1], in[2], a.nrows, out[0], (int)wsm, (int)inb, qmode);
        else if constexpr (B2K_RNE_OPS[OP].wrench) kern<<<grid, B2K_THREADS, smem, st>>>(P, in[0], in[1], in[2], a.nrows, out[0], out[1], (int)wsm, (int)inb, qmode);
        else kern<<<grid, B2K_THREADS, smem, st>>>(P, in[0], in[1], in[2], a.nrows, out[0], out[1], out[2], (int)wsm, (int)inb, qmode);
        b2k_count_launch();
        B2K_CUDA(cudaGetLastError());
        return B2K_OK;
    };
    bool allrev = true;
    for (int j = 0; j < N; j++) allrev = allrev && !P.prismatic[j];
    if (r->mdh) return allrev ? launch(rne_generic_kernel<real, N, true, true, OP>()) : launch(rne_generic_kernel<real, N, true, false, OP>());
    return allrev ? launch(rne_generic_kernel<real, N, false, true, OP>()) : launch(rne_generic_kernel<real, N, false, false, OP>());
}

// The generic kernels of the operations OPS for one dtype, the entry point of the translation unit that instantiates
// them; op is one of OPS (b2k_api.cu picks the unit).
template <typename real, int... OPS>
int rne_generic_launch(const b2k_rne_s *r, int op, const b2k_rne_args &a, cudaStream_t st)
{
    int rc = B2K_ERR_INVALID;
#define B2K_CASE(NN) \
    case NN: ((op == OPS && (rc = rne_generic_launch_op<real, NN, OPS>(r, a, st), true)) || ...); return rc;
    switch (r->n) {
        B2K_CASE(1) B2K_CASE(2) B2K_CASE(3) B2K_CASE(4) B2K_CASE(5)
        B2K_CASE(6) B2K_CASE(7) B2K_CASE(8) B2K_CASE(9) B2K_CASE(10)
    default:
        b2k_set_error("rne: unsupported joint count %d", r->n);
        return B2K_ERR_INVALID;
    }
#undef B2K_CASE
}

// The normal equations of a regressor over a.nrows rows (a.in = q, qd, qdd; grav in a.grav), tau (N, n) of the compute
// type, w the n joint weights; G (p, p), b (p), s (1) fp64 device arrays, p = k n with k parameters per link.  make_y(ca)
// writes the rows of one chunk (ca.in, ca.nrows) into ca.out[0] = Y (ca.nrows, n, p) and returns a b2k_status: the DH
// and the tree regressors share the chunks, the slices and the two reduction kernels.  The caller has checked every
// argument and handles N = 0.
template <typename real, typename MakeY>
int regressor_gram(int n, int p, const b2k_rne_args &a, const void *tau, const double *w, double *G, double *b, double *s,
                   cudaStream_t st, MakeY &&make_y)
{
    if (n > REG_MAX_ROWS) { b2k_set_error("regressor_gram: %d joint rows exceed %d", n, REG_MAX_ROWS); return B2K_ERR_INVALID; }
    const int nt = (p + 1 + REG_TILE - 1) / REG_TILE, npairs = nt * (nt + 1) / 2;
    const long long chunk = a.nrows < REG_CHUNK ? a.nrows : REG_CHUNK;
    // slices: about two blocks of 256 threads per SM, each slice at least 4 k-steps of a full chunk
    const long long kmax = (chunk * n + REG_KB - 1) / REG_KB;
    int slices = (2 * b2k_num_sms() + npairs - 1) / npairs;
    if (slices > kmax / 4) slices = (int)(kmax / 4 > 0 ? kmax / 4 : 1);
    RegWeights W;
    for (int j = 0; j < REG_MAX_ROWS; j++) W.w[j] = j < n ? (w ? w[j] : 1.0) : 0.0;
    const size_t ybytes = ((size_t)chunk * n * p * sizeof(real) + 255) & ~(size_t)255;
    const size_t pbytes = (size_t)slices * npairs * REG_TILE * REG_TILE * sizeof(double);
    b2k_keep_mempool();
    void *scratch = nullptr;
    B2K_CUDA(cudaMallocAsync(&scratch, ybytes + pbytes, st));
    real *Y = (real *)scratch;
    double *part = (double *)((char *)scratch + ybytes);
    int rc = B2K_OK;
    for (long long c0 = 0; c0 < a.nrows && rc == B2K_OK; c0 += chunk) {
        const long long rows = a.nrows - c0 < chunk ? a.nrows - c0 : chunk;
        b2k_rne_args ca = a;
        for (int i = 0; i < 3; i++) ca.in[i] = (const real *)a.in[i] + c0 * n;
        ca.out[0] = Y;
        ca.nrows = rows;
        rc = make_y(ca);
        if (rc) break;
        k_regressor_syrk<real><<<dim3(npairs, slices), 256, 0, st>>>(Y, (const real *)tau + c0 * n, rows * n, n, p, nt, W, part,
                                                                      c0 > 0);
        b2k_count_launch();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) rc = b2k_cuda_fail(e, "k_regressor_syrk launch");
    }
    if (rc == B2K_OK) {
        const int P = p + 1;
        k_regressor_gram_reduce<REG_TILE><<<(P * P + 255) / 256, 256, 0, st>>>(part, slices, npairs, nt, p, G, b, s);
        b2k_count_launch();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) rc = b2k_cuda_fail(e, "k_regressor_gram_reduce launch");
    }
    const cudaError_t e = cudaFreeAsync(scratch, st);
    if (rc == B2K_OK && e != cudaSuccess) rc = b2k_cuda_fail(e, "cudaFreeAsync");
    return rc;
}

// The normal equations of the DH regressor, p = 14 n; b2k_api.cu has checked every argument and handles N = 0.
template <typename real>
int rne_regressor_gram(const b2k_rne_s *r, const b2k_rne_args &a, const void *tau, const double *w, double *G, double *b,
                       double *s, cudaStream_t st)
{
    return regressor_gram<real>(r->n, 14 * r->n, a, tau, w, G, b, s, st, [&](const b2k_rne_args &ca) {
        return rne_generic_launch<real, B2K_GEN_RNE_REGRESSOR>(r, B2K_GEN_RNE_REGRESSOR, ca, st);
    });
}
