// b2k_trig.cuh -- sincos for the chain walk.
//
// CUDA's sincos() is accurate but costs ~100 issued instructions per call in this kernel
// (ncu): its 14 polynomial coefficients are materialised as pairs of
// 32-bit immediates and the quadrant fix-up is a chain of 22 FSEL.  This version does the same
// mathematics -- three-FMA Cody-Waite reduction by pi/2 (exact products thanks to FMA, valid for
// |x| < 105615 like CUDA's own fast path), fdlibm's degree-13/14 minimax kernels on
// [-pi/4, pi/4] (< 1 ulp each), quadrant swap/sign by integer ops -- with every constant read
// from the kernel-parameter constant bank.  Measured max error 1.6 ulp (tests/test_gpu_parity.py::
// test_sincos_accuracy).  Arguments beyond the fast range, infinities and NaNs take CUDA's
// sincos (Payne-Hanek) on a rarely taken branch.
#pragma once

#include "b2k_common.cuh"

#define B2K_MUFU_LIMIT 8.0f

// out-of-line so the seven call sites of an unrolled chain do not each inline Payne-Hanek
// (results are returned BY VALUE: taking the address of the caller's s / c would pin them to
// local memory on the fast path too)
static __device__ __noinline__ double2 b2k_sincos_slow(double x)
{
    double s, c;
    sincos(x, &s, &c);
    return make_double2(s, c);
}
static __device__ __noinline__ float2 b2k_sincos_slow(float x)
{
    float s, c;
    sincosf(x, &s, &c);
    return make_float2(s, c);
}

__device__ __forceinline__ void b2k_sincos(double x, const TrigC<double> &t, double *sp, double *cp)
{
    if (!(fabs(x) < t.fast_limit)) {
        const double2 r = b2k_sincos_slow(x);
        *sp = r.x;
        *cp = r.y;
        return;
    }
    const double tt = fma(x, t.two_over_pi, t.magic);
    const int q = __double2loint(tt);
    const double kd = tt - t.magic;
    double r = fma(-kd, t.pio2_hi, x);
    r = fma(-kd, t.pio2_mid, r);
    r = fma(-kd, t.pio2_lo, r);
    const double z = r * r;
    double ps = fma(t.s[5], z, t.s[4]);
    ps = fma(ps, z, t.s[3]);
    ps = fma(ps, z, t.s[2]);
    ps = fma(ps, z, t.s[1]);
    ps = fma(ps, z, t.s[0]);
    double pc = fma(t.c[5], z, t.c[4]);
    pc = fma(pc, z, t.c[3]);
    pc = fma(pc, z, t.c[2]);
    pc = fma(pc, z, t.c[1]);
    pc = fma(pc, z, t.c[0]);
    const double sn = fma(r * z, ps, r);
    const double cs = fma(z * z, pc, fma(-0.5, z, 1.0));
    // quadrant: n=0 (s,c) ; 1 (c,-s) ; 2 (-s,-c) ; 3 (-c,s)
    const bool swap = q & 1;
    double s = swap ? cs : sn;
    double c = swap ? sn : cs;
    const int sflip = (q & 2) << 30;       // bit 31 if n in {2,3}
    const int cflip = ((q + 1) & 2) << 30; // bit 31 if n in {1,2}
    *sp = __hiloint2double(__double2hiint(s) ^ sflip, __double2loint(s));
    *cp = __hiloint2double(__double2hiint(c) ^ cflip, __double2loint(c));
}

__device__ __forceinline__ void b2k_sincos(float x, const TrigC<float> &t, float *sp, float *cp)
{
    if (!(fabsf(x) < t.fast_limit)) {
        const float2 r = b2k_sincos_slow(x);
        *sp = r.x;
        *cp = r.y;
        return;
    }
    const float tt = fmaf(x, t.two_over_pi, t.magic);
    const int q = __float_as_int(tt);
    const float kd = tt - t.magic;
    float r = fmaf(-kd, t.pio2_hi, x);
    r = fmaf(-kd, t.pio2_mid, r);
    r = fmaf(-kd, t.pio2_lo, r);
    const float z = r * r;
    float ps = fmaf(t.s[2], z, t.s[1]);
    ps = fmaf(ps, z, t.s[0]);
    float pc = fmaf(t.c[2], z, t.c[1]);
    pc = fmaf(pc, z, t.c[0]);
    const float sn = fmaf(r * z, ps, r);
    const float cs = fmaf(z * z, pc, fmaf(-0.5f, z, 1.0f));
    const bool swap = q & 1;
    float s = swap ? cs : sn;
    float c = swap ? sn : cs;
    const int sflip = (q & 2) << 30;
    const int cflip = ((q + 1) & 2) << 30;
    *sp = __int_as_float(__float_as_int(s) ^ sflip);
    *cp = __int_as_float(__float_as_int(c) ^ cflip);
}

// N independent sincos evaluated stage by stage: every coefficient is fetched once and used N
// times, and the N dependency chains interleave (instruction-level parallelism for a kernel that
// runs only ~4 warps per scheduler).
// fp32, any finite angle, no data-dependent path: r = x - 2 pi rint(x / 2 pi) by a two-term Cody-Waite product, then
// sin.approx / cos.approx on |r| <= pi (absolute error 2^-21.4 there; the reduction adds ~|x| 2^-24 relative to a
// period, i.e. nothing below |x| ~ 1e3 and an angle that is itself only known to an ulp beyond).  7 instructions
// per joint.  Used by the IK loop, where a diverging iterate in one lane must not send the whole warp through the
// polynomial path as well as the fast one.
template <int N>
__device__ __forceinline__ void b2k_sincos_batch_reduced(const float *x, float *s, float *c)
{
#pragma unroll
    for (int j = 0; j < N; j++) {
        const float k = rintf(x[j] * 0.15915494309189535f);
        float r = fmaf(-k, 6.2831854820251465f, x[j]);
        r = fmaf(-k, -1.7484555e-7f, r);
        s[j] = __sinf(r);
        c[j] = __cosf(r);
    }
}

template <typename real, int N>
__device__ __forceinline__ void b2k_sincos_batch(const real *x, const TrigC<real> &t, real *s, real *c)
{
    if constexpr (sizeof(real) == 4) {
        // fp32, moderate angles: the special-function unit.  sin.approx / cos.approx reduce by a single multiply with
        // 1/(2 pi), so their absolute error grows with |x| (2^-21.4 + |x| 2^-25): below B2K_MUFU_LIMIT it stays
        // under 7e-7, two orders of magnitude inside the fp32 parity bar (1e-4), for 3 issued instructions per
        // joint instead of 25.  Larger angles take the Cody-Waite + polynomial path below.
        bool all_small = true;
#pragma unroll
        for (int j = 0; j < N; j++) all_small = all_small && (fabsf(x[j]) < B2K_MUFU_LIMIT);
        if (all_small) {
#pragma unroll
            for (int j = 0; j < N; j++) { s[j] = __sinf(x[j]); c[j] = __cosf(x[j]); }
            return;
        }
    }
    bool all_fast = true;
#pragma unroll
    for (int j = 0; j < N; j++) all_fast = all_fast && (fabs(x[j]) < t.fast_limit);
    if (!all_fast) { // rare: huge / non-finite angles somewhere in this row
#pragma unroll
        for (int j = 0; j < N; j++) b2k_sincos(x[j], t, &s[j], &c[j]);
        return;
    }
    real r[N], z[N], ps[N], pc[N];
    int q[N];
#pragma unroll
    for (int j = 0; j < N; j++) {
        const real tt = fma(x[j], t.two_over_pi, t.magic);
        if constexpr (sizeof(real) == 8) q[j] = __double2loint(tt);
        else q[j] = __float_as_int(tt);
        const real kd = tt - t.magic;
        real rr = fma(-kd, t.pio2_hi, x[j]);
        rr = fma(-kd, t.pio2_mid, rr);
        r[j] = fma(-kd, t.pio2_lo, rr);
        z[j] = r[j] * r[j];
    }
    constexpr int D = sizeof(real) == 8 ? 6 : 3; // polynomial terms
#pragma unroll
    for (int j = 0; j < N; j++) { ps[j] = t.s[D - 1]; pc[j] = t.c[D - 1]; }
#pragma unroll
    for (int k = D - 2; k >= 0; k--) {
#pragma unroll
        for (int j = 0; j < N; j++) { ps[j] = fma(ps[j], z[j], t.s[k]); pc[j] = fma(pc[j], z[j], t.c[k]); }
    }
#pragma unroll
    for (int j = 0; j < N; j++) {
        const real sn = fma(r[j] * z[j], ps[j], r[j]);
        const real cs = fma(z[j] * z[j], pc[j], fma((real)-0.5, z[j], (real)1));
        const bool swap = q[j] & 1;
        const real ss = swap ? cs : sn;
        const real cc = swap ? sn : cs;
        const int sflip = (q[j] & 2) << 30;
        const int cflip = ((q[j] + 1) & 2) << 30;
        if constexpr (sizeof(real) == 8) {
            s[j] = __hiloint2double(__double2hiint(ss) ^ sflip, __double2loint(ss));
            c[j] = __hiloint2double(__double2hiint(cc) ^ cflip, __double2loint(cc));
        } else {
            s[j] = __int_as_float(__float_as_int(ss) ^ sflip);
            c[j] = __int_as_float(__float_as_int(cc) ^ cflip);
        }
    }
}
