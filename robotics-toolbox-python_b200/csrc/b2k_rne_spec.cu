// b2k_rne_spec.cu -- run-time compilation and launch of the robot-specialised RNE kernels.
//
// b2k_rne_gen.cpp turns one robot's 24-double link table into straight-line CUDA C for the recursion
// (and for the dynamics fan-outs built on it).  Here that text is wrapped in the tile I/O of the RNE
// kernels (a warp owns 32 rows: cp.async tiles in, one row per lane, results staged and written by one
// TMA bulk copy), compiled for sm_90a with NVRTC the first time a (robot, operation, dtype, gravity
// pattern) is used, loaded through the driver API and launched on the caller's stream.  Both libraries
// are found with dlopen at run time (libnvrtc.so.12 of the CUDA toolkit, libcuda.so.1 of the driver):
// libb2kin.so itself links neither.  When either is missing the
// pre-compiled generic kernels of b2k_rne.cuh serve the call -- still on the GPU; nothing here ever
// computes on the host.  B2K_RNE_SPEC=0 disables the specialised path, B2K_RNE_SPEC=2 turns a failure
// to specialise into an error (tests use it to prove which kernel ran).
#include <cuda.h>
#include <dlfcn.h>
#include <nvrtc.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cmath>

#include <algorithm>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "b2k_rne_gen.h"

namespace {

// ------------------------------------------------------------------ the fixed part of the kernel source
// Macros supplied on the NVRTC command line: REAL, NJ (joints), NC (constant-bank entries), MODE
// (B2K_GEN_*), NIN (input arrays), NOUT (reals written per row), NRES (reals the row function returns),
// PADIN (1: padded input rows, element-wise tile load), MINB (resident blocks per SM to aim for); NOUT2 (only for
// B2K_GEN_RNE_WRENCH: reals per row of a second output array, res[NOUT..NOUT+NOUT2), staged and copied on its own).
// WPB: warps per block of the derivative kernels (kDeriv), chosen from n so that their output stage fits.
const char *kPrologue = R"B2KSRC(
typedef REAL real;
typedef unsigned long long u64;
struct TrigC { real two_over_pi, magic, pio2_hi, pio2_mid, pio2_lo, fast_limit; real s[6]; real c[6]; };
struct SpecP { real C[NC]; real grav[3]; real fext[6]; real offset[NJ]; TrigC trig; };

// 1 where x > 0 (x < 0), else 0: compiles to a SET instruction, so the Coulomb term is two FMAs and no branch
__device__ __forceinline__ real step_pos(real x) { return x > (real)0 ? (real)1 : (real)0; }
__device__ __forceinline__ real step_neg(real x) { return x < (real)0 ? (real)1 : (real)0; }

// sincos of the NJ joint angles as one interleaved batch: three-FMA Cody-Waite reduction by pi/2, fdlibm minimax
// kernels on [-pi/4, pi/4], integer quadrant logic; every coefficient comes from the parameter bank (csrc/b2k_trig.cuh
// is the same code; measured <= 1.6 ulp).  fp32 rows with every |angle| < 8 take the special-function unit.
struct SC { real s, c; };
__device__ __noinline__ SC sincos_slow(real x)
{ // by value: taking the address of the caller's arrays would pin them to local memory on the fast path too
    SC r;
#if REAL_IS_F64
    sincos(x, &r.s, &r.c);
#else
    sincosf(x, &r.s, &r.c);
#endif
    return r;
}
__device__ __forceinline__ void sincos_batch(const real *x, const TrigC &t, real *s, real *c)
{
#if !REAL_IS_F64
    real amax = fabs(x[0]); // one comparison for the whole row (|x| is an operand modifier, max a single instruction)
#pragma unroll
    for (int j = 1; j < NJ; j++) amax = fmax(amax, fabs(x[j]));
    {
        if (amax < 8.0f) {
#pragma unroll
            for (int j = 0; j < NJ; j++) { s[j] = __sinf(x[j]); c[j] = __cosf(x[j]); }
            return;
        }
    }
#endif
#if REAL_IS_F64
    real amax = fabs(x[0]);
#pragma unroll
    for (int j = 1; j < NJ; j++) amax = fmax(amax, fabs(x[j]));
#endif
    if (!(amax < t.fast_limit)) { // rare: huge / non-finite angles somewhere in this row (NaN fails the test too)
#pragma unroll
        for (int j = 0; j < NJ; j++) { const SC r = sincos_slow(x[j]); s[j] = r.s; c[j] = r.c; }
        return;
    }
    real r[NJ], z[NJ], ps[NJ], pc[NJ];
    int q[NJ];
#pragma unroll
    for (int j = 0; j < NJ; j++) {
        const real tt = fma(x[j], t.two_over_pi, t.magic);
#if REAL_IS_F64
        q[j] = __double2loint(tt);
#else
        q[j] = __float_as_int(tt);
#endif
        const real kd = tt - t.magic;
        real rr = fma(-kd, t.pio2_hi, x[j]);
        rr = fma(-kd, t.pio2_mid, rr);
        r[j] = fma(-kd, t.pio2_lo, rr);
        z[j] = r[j] * r[j];
    }
    const int D = REAL_IS_F64 ? 6 : 3;
#pragma unroll
    for (int j = 0; j < NJ; j++) { ps[j] = t.s[D - 1]; pc[j] = t.c[D - 1]; }
#pragma unroll
    for (int k = D - 2; k >= 0; k--) {
#pragma unroll
        for (int j = 0; j < NJ; j++) { ps[j] = fma(ps[j], z[j], t.s[k]); pc[j] = fma(pc[j], z[j], t.c[k]); }
    }
#pragma unroll
    for (int j = 0; j < NJ; j++) {
        const real sn = fma(r[j] * z[j], ps[j], r[j]);
        const real cs = fma(z[j] * z[j], pc[j], fma((real)-0.5, z[j], (real)1));
        const bool swap = q[j] & 1;
        const real ss = swap ? cs : sn;
        const real cc = swap ? sn : cs;
        const int sflip = (q[j] & 2) << 30;
        const int cflip = ((q[j] + 1) & 2) << 30;
#if REAL_IS_F64
        s[j] = __hiloint2double(__double2hiint(ss) ^ sflip, __double2loint(ss));
        c[j] = __hiloint2double(__double2hiint(cc) ^ cflip, __double2loint(cc));
#else
        s[j] = __int_as_float(__float_as_int(ss) ^ sflip);
        c[j] = __int_as_float(__float_as_int(cc) ^ cflip);
#endif
    }
}

// M (NJ x NJ, row-major, symmetric positive definite; only the lower triangle is read) = L D L^T without pivoting, in
// place: L below the diagonal of M, D in d.  The accel kernels, the forward-dynamics integrator and the accel derivatives
// all solve with this one factorisation.
__device__ __forceinline__ void ldlt_factor(real *M, real *d)
{
#pragma unroll
    for (int c = 0; c < NJ; c++) {
        real dc = M[c * NJ + c];
#pragma unroll
        for (int k = 0; k < c; k++) dc = fma(-M[c * NJ + k] * d[k], M[c * NJ + k], dc);
        d[c] = dc;
        const real inv = (real)1 / dc;
#pragma unroll
        for (int r = c + 1; r < NJ; r++) {
            real v = M[r * NJ + c];
#pragma unroll
            for (int k = 0; k < c; k++) v = fma(-M[r * NJ + k] * d[k], M[c * NJ + k], v);
            M[r * NJ + c] = v * inv; // L[r][c]
        }
    }
}

// y <- M^-1 y with the factors of ldlt_factor
__device__ __forceinline__ void ldlt_solve(const real *L, const real *d, real *y)
{
#pragma unroll
    for (int r = 0; r < NJ; r++)
#pragma unroll
        for (int k = 0; k < r; k++) y[r] = fma(-L[r * NJ + k], y[k], y[r]);
#pragma unroll
    for (int r = 0; r < NJ; r++) y[r] = y[r] / d[r];
#pragma unroll
    for (int r = NJ - 1; r >= 0; r--)
#pragma unroll
        for (int k = r + 1; k < NJ; k++) y[r] = fma(-L[k * NJ + r], y[k], y[r]);
}
)B2KSRC";

// the input tiles of the row kernels: 32 rows of NJ reals per array
const char *kTileIn = R"B2KSRC(
#define LDI (PADIN ? (NJ | 1) : NJ)                  /* smem row stride of the input tiles, in reals */
#define IN_BYTES ((32 * LDI * (int)sizeof(real) + 15) & ~15)

__device__ __forceinline__ void load_tile(real *s, const real *g, int lane)
{
#if PADIN
    // padded rows: the exact image would make the one-row-per-lane reads collide on the shared-memory banks
    for (int i = lane; i < 32 * NJ; i += 32) {
        const int r = i / NJ, c = i - r * NJ;
        s[r * LDI + c] = g[i];
    }
#else
    const uint4 *gg = reinterpret_cast<const uint4 *>(g) + lane;
    const unsigned sa = (unsigned)__cvta_generic_to_shared(s) + 16u * (unsigned)lane;
    constexpr int UNITS = (32 * NJ * (int)sizeof(real)) / 16; // 16-byte units in the tile: trip count known at compile time
#pragma unroll
    for (int k = 0; k < (UNITS + 31) / 32; k++)
        if (k * 32 + 32 <= UNITS || lane < UNITS - k * 32)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa + 512u * (unsigned)k), "l"(gg + 32 * k));
#endif
}
)B2KSRC";

const char *kKernel = R"B2KSRC(
#define OUT_BYTES (32 * NOUT * (int)sizeof(real))
#ifndef NOUT2
#define NOUT2 0
#endif
#define NBUF (TPW > 1 ? 2 : 1)                        /* input buffers per warp */
#define WARP_BYTES (NBUF * NIN * IN_BYTES + OUT_BYTES + 32 * NOUT2 * (int)sizeof(real))

// A warp owns TPW consecutive tiles of 32 rows (one-shot grid of full tiles; the ragged tail of a batch goes to the
// generic kernel).  The input tiles are double-buffered: the cp.async loads of tile t+1 are issued before tile t is
// computed, so a warp always has a tile's worth of reads in flight -- with one tile per warp and 16-20 resident warps
// per SM the kernel was latency-bound (ncu: long-scoreboard the top stall, FP64 pipe 62 % busy).
extern "C" __global__ void __launch_bounds__(128, MINB)
k_rne_spec(const __grid_constant__ SpecP P, const real *__restrict__ in0, const real *__restrict__ in1,
           const real *__restrict__ in2, real *__restrict__ out,
#if NOUT2
           real *__restrict__ out2,
#endif
           long long ntiles)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long tile0 = ((long long)blockIdx.x * 4 + warp) * TPW;
    if (tile0 >= ntiles) return;
    unsigned char *wb = smem + (size_t)warp * WARP_BYTES;
    real *so = reinterpret_cast<real *>(wb + NBUF * NIN * IN_BYTES);
    auto load = [&](long long tile, int buf) {
        unsigned char *b = wb + (size_t)buf * NIN * IN_BYTES;
        const size_t row0 = (size_t)tile * 32;
        load_tile(reinterpret_cast<real *>(b), in0 + row0 * NJ, lane);
        if (NIN >= 2) load_tile(reinterpret_cast<real *>(b + IN_BYTES), in1 + row0 * NJ, lane);
        if (NIN >= 3) load_tile(reinterpret_cast<real *>(b + 2 * IN_BYTES), in2 + row0 * NJ, lane);
#if !PADIN
        asm volatile("cp.async.commit_group;\n" ::: "memory");
#endif
    };
    load(tile0, 0);
#pragma unroll 1
    for (int t = 0; t < TPW; t++) {
        const long long tile = tile0 + t;
        if (tile >= ntiles) break;
        const bool more = (t + 1 < TPW) && (tile + 1 < ntiles);
        if (more) load(tile + 1, (t + 1) & (NBUF - 1));
#if !PADIN
        if (more) asm volatile("cp.async.wait_group 1;\n" ::: "memory");
        else asm volatile("cp.async.wait_group 0;\n" ::: "memory");
#endif
        __syncwarp();
        const unsigned char *b = wb + (size_t)(t & (NBUF - 1)) * NIN * IN_BYTES;
        const real *s0 = reinterpret_cast<const real *>(b);
        const real *s1 = reinterpret_cast<const real *>(b + IN_BYTES);
        const real *s2 = reinterpret_cast<const real *>(b + 2 * IN_BYTES);
        real th[NJ], st[NJ], ct[NJ], a1[NJ], a2[NJ];
#pragma unroll
        for (int j = 0; j < NJ; j++) {
            th[j] = s0[lane * LDI + j] + P.offset[j];
            a1[j] = NIN >= 2 ? s1[lane * LDI + j] : (real)0;
            a2[j] = NIN >= 3 ? s2[lane * LDI + j] : (real)0;
        }
        sincos_batch(th, P.trig, st, ct);
        real res[NRES];
        rne_row(P.C, P.grav, P.fext, st, ct, th, a1, a2, res);
#if MODE == 5
        // accel: res = [M (NJ x NJ, row i = torques for a unit acceleration of joint i) | torque - rne(q, qd, 0)].
        // M is the joint-space inertia matrix (symmetric positive definite): LDL^T without pivoting, in registers.
        real d[NJ];
        ldlt_factor(res, d);
        real *y = res + NJ * NJ;
        ldlt_solve(res, d, y);
        const real *o = y;
#else
        const real *o = res;
#endif
        // the previous tile's bulk copy must have finished READING the stage before it is overwritten
        if (t > 0) {
            if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            __syncwarp();
        }
#pragma unroll
        for (int k = 0; k < NOUT; k++) so[lane * NOUT + k] = o[k];
#if NOUT2
        real *so2 = so + 32 * NOUT; // the second output's tile, right behind the first (a multiple of 16 bytes)
#pragma unroll
        for (int k = 0; k < NOUT2; k++) so2[lane * NOUT2 + k] = o[NOUT + k];
#endif
        // the staged tile is the exact image of the output block: one TMA bulk copy (shared -> global) by lane 0
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) {
            const unsigned ss = (unsigned)__cvta_generic_to_shared(so);
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(out + (size_t)tile * 32 * NOUT), "r"(ss),
                         "r"((unsigned)OUT_BYTES) : "memory");
#if NOUT2
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(out2 + (size_t)tile * 32 * NOUT2),
                         "r"((unsigned)__cvta_generic_to_shared(so2)), "r"((unsigned)(32 * NOUT2 * sizeof(real))) : "memory");
#endif
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); // the copies read this warp's shared memory
}
)B2KSRC";


// ------------------------------------------------------------------ derivatives of the dynamics of a tree (MODE 7, 8)
// A row writes 2 (RNE_DERIV: dtau_dq, dtau_dqd) or 3 (ACCEL_DERIV: dqdd_dq, dqdd_dqd, dqdd_dtau) blocks of NJ x NJ reals.
// The generated derivative row stores its columns straight into the warp's shared stage, one exact-image n x n tile per
// output (32 rows), copied out by one TMA bulk copy each; the number of warps per block (WPB) is chosen from n so that
// the stage fits (fp64 n = 16, three outputs: 197 KB for one warp).
const char *kDeriv = R"B2KSRC(
#define NSQ (NJ * NJ)
#define NBLK (MODE == 8 ? 3 : 2)
#define BLK_BYTES (32 * NSQ * (int)sizeof(real))
#define WARP_BYTES (NIN * IN_BYTES + NBLK * BLK_BYTES)

extern "C" __global__ void __launch_bounds__(32 * WPB, MINB)
k_rne_deriv_spec(const __grid_constant__ SpecP P, const real *__restrict__ in0, const real *__restrict__ in1,
                 const real *__restrict__ in2, real *__restrict__ out0, real *__restrict__ out1, real *__restrict__ out2,
                 long long ntiles)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long tile = (long long)blockIdx.x * WPB + warp;
    if (tile >= ntiles) return;
    unsigned char *wb = smem + (size_t)warp * WARP_BYTES;
    real *so = reinterpret_cast<real *>(wb + NIN * IN_BYTES);
    const size_t row0 = (size_t)tile * 32;
    load_tile(reinterpret_cast<real *>(wb), in0 + row0 * NJ, lane);
    load_tile(reinterpret_cast<real *>(wb + IN_BYTES), in1 + row0 * NJ, lane);
    load_tile(reinterpret_cast<real *>(wb + 2 * IN_BYTES), in2 + row0 * NJ, lane);
#if !PADIN
    asm volatile("cp.async.commit_group;\n" ::: "memory");
    asm volatile("cp.async.wait_group 0;\n" ::: "memory");
#endif
    __syncwarp();
    const real *s0 = reinterpret_cast<const real *>(wb);
    const real *s1 = reinterpret_cast<const real *>(wb + IN_BYTES);
    const real *s2 = reinterpret_cast<const real *>(wb + 2 * IN_BYTES);
    real th[NJ], st[NJ], ct[NJ], a1[NJ], a2[NJ];
#pragma unroll
    for (int j = 0; j < NJ; j++) {
        th[j] = s0[lane * LDI + j] + P.offset[j];
        a1[j] = s1[lane * LDI + j];
        a2[j] = s2[lane * LDI + j];
    }
    sincos_batch(th, P.trig, st, ct);
    real *d0 = so + lane * NSQ, *d1 = so + 32 * NSQ + lane * NSQ;
#if MODE == 8
    // qdd* = M^-1 (torque - rne(q, qd, 0)) as accel computes it; dqdd_dtau = M^-1 from the same factorisation, staged
    // before the derivative row so that the factors are dead while it runs; then the derivatives of rne(q, qd, qdd*)
    // with qdd* held fixed, mapped in the stage: dqdd_dx = -M^-1 dtau_dx
    real *d2 = so + 64 * NSQ + lane * NSQ, qdd[NJ];
    {
        real res[NJ * NJ + NJ], d[NJ];
        rne_row(P.C, P.grav, P.fext, st, ct, th, a1, a2, res);
        ldlt_factor(res, d);
        ldlt_solve(res, d, res + NSQ);
#pragma unroll
        for (int i = 0; i < NJ; i++) qdd[i] = res[NSQ + i];
#pragma unroll 1
        for (int c = 0; c < NJ; c++) {
            real y[NJ];
#pragma unroll
            for (int i = 0; i < NJ; i++) y[i] = (real)(i == c);
            ldlt_solve(res, d, y);
#pragma unroll
            for (int i = 0; i < NJ; i++) d2[i * NJ + c] = y[i];
        }
    }
    rne_deriv_row(P.C, P.grav, P.fext, st, ct, th, a1, qdd, d0, d1);
#pragma unroll 1
    for (int k = 0; k < 2 * NJ; k++) {
        real *blk = k < NJ ? d0 : d1;
        const int c = k < NJ ? k : k - NJ;
        real x[NJ];
#pragma unroll
        for (int i = 0; i < NJ; i++) x[i] = blk[i * NJ + c];
#pragma unroll
        for (int i = 0; i < NJ; i++) {
            real y = (real)0;
#pragma unroll
            for (int j = 0; j < NJ; j++) y = fma(-d2[i * NJ + j], x[j], y);
            blk[i * NJ + c] = y;
        }
    }
#else
    rne_deriv_row(P.C, P.grav, P.fext, st, ct, th, a1, a2, d0, d1);
#endif
    // the staged tiles are the exact images of the output blocks: one TMA bulk copy (shared -> global) each, by lane 0
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncwarp();
    if (lane == 0) {
        real *outs[3] = {out0, out1, out2};
#pragma unroll
        for (int b = 0; b < NBLK; b++)
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(outs[b] + row0 * NSQ),
                         "r"((unsigned)__cvta_generic_to_shared(so + b * 32 * NSQ)), "r"((unsigned)BLK_BYTES) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); // the copies read this warp's shared memory
    }
}
)B2KSRC";

// ------------------------------------------------------------------ the dynamics regressor of a tree (MODE 10)
// A row of Y is NJ joint rows of 10 NJ reals (20 KB at n = 16 in fp64), too large to stage 32 whole rows per warp.  The
// generated rne_regressor_row(..., i, y) writes joint row i of one row; the warp stages joint row i of its 32 rows in a
// slab (odd row stride: the one-row-per-lane writes are free of bank conflicts) and drains it before the next joint row,
// consecutive lanes on consecutive reals of Y.  WPB warps per block as fit the shared memory, up to 4.
const char *kReg = R"B2KSRC(
#define ROWY (10 * NJ)                                  /* reals of one joint row of Y */
#define LDY (ROWY | 1)                                  /* slab row stride, in reals */
#define SLAB_BYTES ((32 * LDY * (int)sizeof(real) + 15) & ~15)
#define WARP_BYTES (NIN * IN_BYTES + SLAB_BYTES)

extern "C" __global__ void __launch_bounds__(32 * WPB, MINB)
k_rne_regressor_spec(const __grid_constant__ SpecP P, const real *__restrict__ in0, const real *__restrict__ in1,
                     const real *__restrict__ in2, real *__restrict__ out, long long ntiles)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long tile = (long long)blockIdx.x * WPB + warp;
    if (tile >= ntiles) return;
    unsigned char *wb = smem + (size_t)warp * WARP_BYTES;
    real *slab = reinterpret_cast<real *>(wb + NIN * IN_BYTES);
    const size_t row0 = (size_t)tile * 32;
    load_tile(reinterpret_cast<real *>(wb), in0 + row0 * NJ, lane);
    load_tile(reinterpret_cast<real *>(wb + IN_BYTES), in1 + row0 * NJ, lane);
    load_tile(reinterpret_cast<real *>(wb + 2 * IN_BYTES), in2 + row0 * NJ, lane);
#if !PADIN
    asm volatile("cp.async.commit_group;\n" ::: "memory");
    asm volatile("cp.async.wait_group 0;\n" ::: "memory");
#endif
    __syncwarp();
    const real *s0 = reinterpret_cast<const real *>(wb);
    const real *s1 = reinterpret_cast<const real *>(wb + IN_BYTES);
    const real *s2 = reinterpret_cast<const real *>(wb + 2 * IN_BYTES);
    real th[NJ], st[NJ], ct[NJ], a1[NJ], a2[NJ];
#pragma unroll
    for (int j = 0; j < NJ; j++) {
        th[j] = s0[lane * LDI + j] + P.offset[j];
        a1[j] = s1[lane * LDI + j];
        a2[j] = s2[lane * LDI + j];
    }
    sincos_batch(th, P.trig, st, ct);
    real *gt = out + row0 * (size_t)(NJ * ROWY);
#pragma unroll 1
    for (int i = 0; i < NJ; i++) {
        rne_regressor_row(P.C, P.grav, P.fext, st, ct, th, a1, a2, i, slab + lane * LDY);
        __syncwarp();
        real *g = gt + i * ROWY; // joint row i of the tile's first row; the tile's rows are NJ * ROWY apart
#pragma unroll 4
        for (int e = lane; e < 32 * ROWY; e += 32) {
            const int r = e / ROWY, c = e - r * ROWY;
            g[(size_t)r * (NJ * ROWY) + c] = slab[r * LDY + c];
        }
        __syncwarp();
    }
}
)B2KSRC";

// ------------------------------------------------------------------ forward-dynamics integrator (DynamicsMixin.fdyn)
// The reference integrates ONE state with scipy's RK45, calling accel() -- n + 1 Python rne loops and a numpy solve --
// for every stage (Dynamics.py:185-422).  Here one lane integrates one trajectory of an ensemble entirely on the device:
// Dormand-Prince 5(4) with scipy's step control restated (scipy/integrate/_ivp/rk.py: select_initial_step, the RMS error
// norm against atol + rtol max(|y|, |y_new|), SAFETY 0.9, factors in [0.2, 10], no growth after a rejection), the
// acceleration of every stage from the robot-specialised recursion (mode "accel": inertia rows + bias torque, LDL^T).
// Torque input: none, a constant vector, or a joint-space PD law -- a Python callable cannot run here (DHRobot.fdyn
// takes that route through scipy on the host, with this library's batched accel as the right-hand side).
const char *kFdyn = R"B2KSRC(
struct FdynP {
    real T, rtol, atol, max_step, first_step, dt;
    real kp[NJ], kd[NJ], qstar[NJ], tau[NJ];
    int torque_mode; // 0 none, 1 constant (tau), 2 per-trajectory constant (tau_rows), 3 PD: kp (qstar - q) - kd qd
    int grid;        // 0: store the accepted steps (capacity M per trajectory); 1: store the uniform grid k dt (M samples)
    int M;
};

__device__ __forceinline__ void fd_accel(const SpecP &P, const FdynP &F, const real *tau_row, const real *y, real *qdd)
{
    real th[NJ], st[NJ], ct[NJ], tq[NJ], res[NJ * NJ + NJ];
#pragma unroll
    for (int j = 0; j < NJ; j++) {
        th[j] = y[j] + P.offset[j];
        real t = 0;
        if (F.torque_mode == 1) t = F.tau[j];
        else if (F.torque_mode == 2) t = tau_row[j];
        else if (F.torque_mode == 3) t = F.kp[j] * (F.qstar[j] - y[j]) - F.kd[j] * y[NJ + j];
        tq[j] = t;
    }
    sincos_batch(th, P.trig, st, ct);
    rne_row(P.C, P.grav, P.fext, st, ct, th, y + NJ, tq, res);
    real d[NJ];
    ldlt_factor(res, d);
    real *x = res + NJ * NJ;
    ldlt_solve(res, d, x);
#pragma unroll
    for (int j = 0; j < NJ; j++) qdd[j] = x[j];
}

// f(t, y) = [qd, accel(q, qd, tau(t, q, qd))]
__device__ __noinline__ void fd_rhs(const SpecP &P, const FdynP &F, const real *tau_row, const real *y, real *f)
{
#pragma unroll
    for (int j = 0; j < NJ; j++) f[j] = y[NJ + j];
    fd_accel(P, F, tau_row, y, f + NJ);
}

__device__ __forceinline__ real fd_rms(const real *v, const real *scale)
{
    real s = 0;
    for (int i = 0; i < 2 * NJ; i++) { const real e = v[i] / scale[i]; s = fma(e, e, s); }
    return sqrt(s / (real)(2 * NJ));
}

extern "C" __global__ void __launch_bounds__(64)
k_fdyn(const __grid_constant__ SpecP P, const __grid_constant__ FdynP F, const real *__restrict__ q0, const real *__restrict__ qd0,
       const real *__restrict__ tau_rows, real *__restrict__ out_t, real *__restrict__ out_q, real *__restrict__ out_qd,
       int *__restrict__ out_count, int *__restrict__ out_status, long long ntraj)
{
    const long long tr = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (tr >= ntraj) return;
    constexpr int NS = 2 * NJ;
    // Dormand-Prince tableau (scipy RK45)
    const real C2 = (real)(1.0 / 5), C3 = (real)(3.0 / 10), C4 = (real)(4.0 / 5), C5 = (real)(8.0 / 9);
    const real A[6][5] = {{0, 0, 0, 0, 0},
                          {(real)(1.0 / 5), 0, 0, 0, 0},
                          {(real)(3.0 / 40), (real)(9.0 / 40), 0, 0, 0},
                          {(real)(44.0 / 45), (real)(-56.0 / 15), (real)(32.0 / 9), 0, 0},
                          {(real)(19372.0 / 6561), (real)(-25360.0 / 2187), (real)(64448.0 / 6561), (real)(-212.0 / 729), 0},
                          {(real)(9017.0 / 3168), (real)(-355.0 / 33), (real)(46732.0 / 5247), (real)(49.0 / 176), (real)(-5103.0 / 18656)}};
    const real Bc[6] = {(real)(35.0 / 384), 0, (real)(500.0 / 1113), (real)(125.0 / 192), (real)(-2187.0 / 6784), (real)(11.0 / 84)};
    const real E[7] = {(real)(-71.0 / 57600), 0, (real)(71.0 / 16695), (real)(-71.0 / 1920), (real)(17253.0 / 339200), (real)(-22.0 / 525), (real)(1.0 / 40)};
    const real Cn[6] = {0, C2, C3, C4, C5, 1};
    (void)Cn; // the torque laws served here do not depend on t explicitly
    const real *tau_row = tau_rows ? tau_rows + tr * NJ : nullptr;
    real y[NS], yn[NS], K[7][NS], scale[NS], tmp[NS];
    for (int j = 0; j < NJ; j++) { y[j] = q0[tr * NJ + j]; y[NJ + j] = qd0 ? qd0[tr * NJ + j] : (real)0; }
    real t = 0;
    fd_rhs(P, F, tau_row, y, K[0]);
    // ---- select_initial_step
    real h_abs;
    if (F.first_step > 0) h_abs = F.first_step;
    else {
        for (int i = 0; i < NS; i++) scale[i] = F.atol + fabs(y[i]) * F.rtol;
        const real d0 = fd_rms(y, scale), d1 = fd_rms(K[0], scale);
        real h0 = (d0 < (real)1e-5 || d1 < (real)1e-5) ? (real)1e-6 : (real)0.01 * d0 / d1;
        h0 = fmin(h0, F.T);
        for (int i = 0; i < NS; i++) yn[i] = fma(h0, K[0][i], y[i]);
        fd_rhs(P, F, tau_row, yn, K[1]);
        for (int i = 0; i < NS; i++) tmp[i] = K[1][i] - K[0][i];
        const real d2 = fd_rms(tmp, scale) / h0;
        const real h1 = (d1 <= (real)1e-15 && d2 <= (real)1e-15) ? fmax((real)1e-6, h0 * (real)1e-3) : pow((real)0.01 / fmax(d1, d2), (real)0.2);
        h_abs = fmin(fmin((real)100 * h0, h1), fmin(F.T, F.max_step));
    }
    // ---- output of the initial state
    const size_t obase = (size_t)tr * F.M;
    int count = 0, status = 0;
    auto emit = [&](real tt, const real *yy) {
        if (count < F.M) {
            out_t[obase + count] = tt;
            for (int j = 0; j < NJ; j++) { out_q[(obase + count) * NJ + j] = yy[j]; out_qd[(obase + count) * NJ + j] = yy[NJ + j]; }
        }
        count++;
    };
    int next_grid = 0;
    if (F.grid) { emit(0, y); next_grid = 1; }
    else emit(0, y);
    // ---- the stepping loop of RungeKutta._step_impl
    while (t < F.T) {
        const real min_step = (real)10 * (nextafter(t, (real)1e300) - t);
        if (h_abs > F.max_step) h_abs = F.max_step;
        else if (h_abs < min_step) h_abs = min_step;
        bool accepted = false, rejected = false;
        real tn = t, h = 0;
        while (!accepted) {
            if (h_abs < min_step) { status = 1; break; } // step size too small
            h = h_abs;
            tn = t + h;
            if (tn - F.T > 0) tn = F.T;
            h = tn - t;
            h_abs = fabs(h);
            // rk_step
            for (int s = 1; s < 6; s++) {
                for (int i = 0; i < NS; i++) {
                    real dy = 0;
                    for (int k = 0; k < s; k++) dy += K[k][i] * A[s][k];
                    yn[i] = y[i] + dy * h;
                }
                fd_rhs(P, F, tau_row, yn, K[s]);
            }
            for (int i = 0; i < NS; i++) {
                real dy = 0;
                for (int k = 0; k < 6; k++) dy += K[k][i] * Bc[k];
                yn[i] = y[i] + h * dy;
            }
            fd_rhs(P, F, tau_row, yn, K[6]);
            for (int i = 0; i < NS; i++) {
                scale[i] = F.atol + fmax(fabs(y[i]), fabs(yn[i])) * F.rtol;
                real e = 0;
                for (int k = 0; k < 7; k++) e += K[k][i] * E[k];
                tmp[i] = e * h;
            }
            const real err = fd_rms(tmp, scale);
            if (err < 1) {
                real factor = err == 0 ? (real)10 : fmin((real)10, (real)0.9 * pow(err, (real)-0.2));
                if (rejected) factor = fmin((real)1, factor);
                h_abs *= factor;
                accepted = true;
            } else {
                h_abs *= fmax((real)0.2, (real)0.9 * pow(err, (real)-0.2));
                rejected = true;
            }
        }
        if (!accepted) break;
        if (F.grid) { // linear interpolation onto k dt, as the reference does with interp1d (Dynamics.py:371-377)
            while (next_grid < F.M && (real)next_grid * F.dt <= tn) {
                const real tg = (real)next_grid * F.dt, a = (tg - t) / (tn - t);
                for (int i = 0; i < NS; i++) tmp[i] = y[i] + a * (yn[i] - y[i]);
                emit(tg, tmp);
                next_grid++;
            }
        } else emit(tn, yn);
        t = tn;
        for (int i = 0; i < NS; i++) { y[i] = yn[i]; K[0][i] = K[6][i]; }
    }
    // np.arange(0, T, dt) can end on T itself (T = 2.1, dt = 0.3), and k dt in `real` may round above T (fp32): the
    // samples not yet written are the state at T
    if (F.grid && status == 0)
        for (; next_grid < F.M; next_grid++) emit((real)next_grid * F.dt, y);
    out_count[tr] = count;
    out_status[tr] = status | (count > F.M ? 2 : 0); // 2: more accepted steps than the capacity M
}
)B2KSRC";

// ------------------------------------------------------------------ fixed-step RK4 rollouts (DHRobot.rollout, Robot.rollout)
// One lane integrates one trajectory, as k_fdyn does.  Each stage is one ACCEL row (rne_row) and its LDL^T solve; with
// SENS (the ACCEL_DERIV program) also M^-1 from the same factors, the derivative row at qdd* mapped by -M^-1, and the
// stage's column of the chain rule dk_i = J_f (e + c dt dk_{i-1}) (+ [0; M^-1] for the torque columns), J_f = [[0, I],
// [dqdd_dq, dqdd_dqd]], whose upper half is a copy.  The per-lane working set (dk_{i-1} and the sums of the stages, 6 n^2
// reals each, and three n x n blocks) lives in local memory.  The 6 n^2 reals of A_k | B_k leave through a per-warp slab of
// 32 lanes x CH reals: the warp writes one lane's CH consecutive reals per store instruction, so every store is coalesced
// at every n, where a stage of whole blocks (32 x 6 n^2 reals) would not fit the shared memory from n = 13 (fp64) on.
// Both programs run the same value path (compiled without FMA contraction), so their states are bit-identical.
const char *kRollout = R"B2KSRC(
#define NS (2 * NJ)
#define NSQ (NJ * NJ)
#define NSENS (6 * NSQ)  /* reals of A_k (2n x 2n) followed by B_k (2n x n) */
#define CH 32            /* reals per lane of one drain of the slab */

struct RollP { real h2, h, h6; int K; long long tau_stride; };

extern "C" __global__ void __launch_bounds__(64)
k_rollout(const __grid_constant__ SpecP P, const __grid_constant__ RollP R, const real *__restrict__ q0, const real *__restrict__ qd0,
          const real *__restrict__ tau, real *__restrict__ oq, real *__restrict__ oqd, real *__restrict__ oA, real *__restrict__ oB,
          long long ntraj)
{
    const long long tr = (long long)blockIdx.x * 64 + threadIdx.x;
    if (tr - (threadIdx.x & 31) >= ntraj) return; // a warp with no trajectory (the drains synchronise within a warp only)
    const bool live = tr < ntraj; // dead lanes integrate the zero state and store nothing: the drains need the whole warp
    const long long trc = live ? tr : 0;
    real x[NS];
#pragma unroll
    for (int j = 0; j < NJ; j++) {
        x[j] = live ? q0[trc * NJ + j] : (real)0;
        x[NJ + j] = live && qd0 ? qd0[trc * NJ + j] : (real)0;
    }
    auto store = [&](int k) {
        if (!live) return;
        const size_t o = ((size_t)tr * (R.K + 1) + k) * NJ;
#pragma unroll
        for (int j = 0; j < NJ; j++) { oq[o + j] = x[j]; oqd[o + j] = x[NJ + j]; }
    };
    store(0);
#if SENS
    __shared__ real slab[2][32 * (CH + 1)];
    const int lane = threadIdx.x & 31;
    real *sl = slab[threadIdx.x >> 5];
    const long long tw = tr - lane; // the warp's first trajectory
    // dk_{i-1} and the weighted sum of the stages, both laid out as A_k | B_k: column c < 2n of x at [i * 2n + c], column
    // c of tau at [4 n^2 + i * n + c]
    real Pk[NSENS], acc[NSENS], Dq[NSQ], Dqd[NSQ], Mi[NSQ];
#endif
    const real *tbase = tau + trc * R.tau_stride;
#pragma unroll 1
    for (int k = 0; k < R.K; k++) {
        real tq[NJ], ks[NS], kp[NS];
#pragma unroll
        for (int j = 0; j < NJ; j++) tq[j] = tbase[(size_t)k * NJ + j];
#pragma unroll 1
        for (int s = 0; s < 4; s++) {
            const real c = s == 0 ? (real)0 : s == 3 ? R.h : R.h2;
            real xs[NS];
#pragma unroll
            for (int i = 0; i < NS; i++) xs[i] = s == 0 ? x[i] : fma(c, kp[i], x[i]);
            real th[NJ], st[NJ], ct[NJ], res[NSQ + NJ], d[NJ];
#pragma unroll
            for (int j = 0; j < NJ; j++) th[j] = xs[j] + P.offset[j];
            sincos_batch(th, P.trig, st, ct);
            rne_row(P.C, P.grav, P.fext, st, ct, th, xs + NJ, tq, res);
            ldlt_factor(res, d);
            ldlt_solve(res, d, res + NSQ);
            real kn[NS];
#pragma unroll
            for (int j = 0; j < NJ; j++) { kn[j] = xs[NJ + j]; kn[NJ + j] = res[NSQ + j]; }
#if SENS
#pragma unroll 1
            for (int cc = 0; cc < NJ; cc++) { // M^-1, column by column, before the derivative row: the factors die here
                real y[NJ];
#pragma unroll
                for (int i = 0; i < NJ; i++) y[i] = (real)(i == cc);
                ldlt_solve(res, d, y);
#pragma unroll
                for (int i = 0; i < NJ; i++) Mi[i * NJ + cc] = y[i];
            }
            rne_deriv_row(P.C, P.grav, P.fext, st, ct, th, xs + NJ, kn + NJ, Dq, Dqd);
#pragma unroll 1
            for (int cc = 0; cc < NS; cc++) { // dqdd_dx = -M^-1 dtau_dx, in place
                real *blk = cc < NJ ? Dq : Dqd;
                const int cj = cc < NJ ? cc : cc - NJ;
                real v[NJ];
#pragma unroll
                for (int i = 0; i < NJ; i++) v[i] = blk[i * NJ + cj];
#pragma unroll
                for (int i = 0; i < NJ; i++) {
                    real y = (real)0;
#pragma unroll
                    for (int j = 0; j < NJ; j++) y = fma(-Mi[i * NJ + j], v[j], y);
                    blk[i * NJ + cj] = y;
                }
            }
            const real w = s == 0 || s == 3 ? (real)1 : (real)2;
#pragma unroll 1
            for (int col = 0; col < NS + NJ; col++) {
                const bool xcol = col < NS;
                const int base = xcol ? col : 4 * NSQ + col - NS, ld = xcol ? NS : NJ;
                real sv[NS]; // the stage state's derivative along this column: e_col (x only) + c dt dk_{i-1}
#pragma unroll
                for (int i = 0; i < NS; i++) {
                    const real e = (real)(xcol && i == col);
                    sv[i] = s == 0 ? e : fma(c, Pk[base + i * ld], e);
                }
                real nv[NS];
#pragma unroll
                for (int r = 0; r < NJ; r++) {
                    nv[r] = sv[NJ + r];
                    real y = xcol ? (real)0 : Mi[r * NJ + col - NS];
#pragma unroll
                    for (int m = 0; m < NJ; m++) y = fma(Dq[r * NJ + m], sv[m], y);
#pragma unroll
                    for (int m = 0; m < NJ; m++) y = fma(Dqd[r * NJ + m], sv[NJ + m], y);
                    nv[NJ + r] = y;
                }
#pragma unroll
                for (int i = 0; i < NS; i++) {
                    Pk[base + i * ld] = nv[i];
                    acc[base + i * ld] = s == 0 ? nv[i] : fma(w, nv[i], acc[base + i * ld]);
                }
            }
#endif
#pragma unroll
            for (int i = 0; i < NS; i++) {
                ks[i] = s == 0 ? kn[i] : fma(s == 3 ? (real)1 : (real)2, kn[i], ks[i]);
                kp[i] = kn[i];
            }
        }
#pragma unroll
        for (int i = 0; i < NS; i++) x[i] = fma(R.h6, ks[i], x[i]);
        store(k + 1);
#if SENS
        // A_k = I + dt/6 (dk1 + 2 dk2 + 2 dk3 + dk4), B_k = dt/6 (...), drained CH reals per lane at a time
#pragma unroll 1
        for (int c0 = 0; c0 < NSENS; c0 += CH) {
#pragma unroll 4
            for (int e = 0; e < CH; e++) {
                const int i = c0 + e;
                if (i < NSENS) sl[lane * (CH + 1) + e] = fma(R.h6, acc[i], (real)(i < 4 * NSQ && i % (NS + 1) == 0));
            }
            __syncwarp();
#pragma unroll 4
            for (int r = 0; r < 32; r++) {
                const int i = c0 + lane;
                if (i < NSENS && tw + r < ntraj) {
                    const size_t blk = (size_t)(tw + r) * R.K + k;
                    const real v = sl[r * (CH + 1) + lane];
                    if (i < 4 * NSQ) oA[blk * (4 * NSQ) + i] = v;
                    else oB[blk * (2 * NSQ) + i - 4 * NSQ] = v;
                }
            }
            __syncwarp();
        }
#endif
    }
}
)B2KSRC";

// ------------------------------------------------------------------ dynamic loading of NVRTC and the driver API
struct Nvrtc {
    void *h = nullptr;
    nvrtcResult (*CreateProgram)(nvrtcProgram *, const char *, const char *, int, const char *const *, const char *const *);
    nvrtcResult (*CompileProgram)(nvrtcProgram, int, const char *const *);
    nvrtcResult (*GetCUBINSize)(nvrtcProgram, size_t *);
    nvrtcResult (*GetCUBIN)(nvrtcProgram, char *);
    nvrtcResult (*GetProgramLogSize)(nvrtcProgram, size_t *);
    nvrtcResult (*GetProgramLog)(nvrtcProgram, char *);
    nvrtcResult (*DestroyProgram)(nvrtcProgram *);
    const char *(*GetErrorString)(nvrtcResult);
    std::string why;
};
struct Driver {
    void *h = nullptr;
    CUresult (*ModuleLoadData)(CUmodule *, const void *);
    CUresult (*ModuleGetFunction)(CUfunction *, CUmodule, const char *);
    CUresult (*ModuleUnload)(CUmodule);
    CUresult (*LaunchKernel)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, CUstream, void **, void **);
    CUresult (*FuncSetAttribute)(CUfunction, CUfunction_attribute, int);
    CUresult (*FuncGetAttribute)(int *, CUfunction_attribute, CUfunction);
    CUresult (*GetErrorString)(CUresult, const char **);
    std::string why;
};

template <typename F>
bool sym(void *h, const char *name, F &fn, std::string &why)
{
    fn = reinterpret_cast<F>(dlsym(h, name));
    if (!fn) { why = std::string("symbol ") + name + " not found"; return false; }
    return true;
}

Nvrtc *nvrtc()
{
    static Nvrtc N;
    static std::once_flag once;
    std::call_once(once, [] {
        std::vector<std::string> cands;
        if (const char *e = getenv("B2K_NVRTC_PATH")) cands.push_back(e);
        for (const char *n : {"libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so"})
            cands.push_back(n);
        for (const std::string &c : cands) {
            N.h = dlopen(c.c_str(), RTLD_NOW | RTLD_LOCAL);
            if (N.h) break;
        }
        if (!N.h) { N.why = "libnvrtc.so.12 not found (set B2K_NVRTC_PATH)"; return; }
        bool ok = sym(N.h, "nvrtcCreateProgram", N.CreateProgram, N.why) && sym(N.h, "nvrtcCompileProgram", N.CompileProgram, N.why) &&
                  sym(N.h, "nvrtcGetCUBINSize", N.GetCUBINSize, N.why) && sym(N.h, "nvrtcGetCUBIN", N.GetCUBIN, N.why) &&
                  sym(N.h, "nvrtcGetProgramLogSize", N.GetProgramLogSize, N.why) && sym(N.h, "nvrtcGetProgramLog", N.GetProgramLog, N.why) &&
                  sym(N.h, "nvrtcDestroyProgram", N.DestroyProgram, N.why) && sym(N.h, "nvrtcGetErrorString", N.GetErrorString, N.why);
        if (!ok) { dlclose(N.h); N.h = nullptr; }
    });
    return &N;
}

Driver *driver()
{
    static Driver D;
    static std::once_flag once;
    std::call_once(once, [] {
        D.h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_LOCAL);
        if (!D.h) { D.why = "libcuda.so.1 not found"; return; }
        bool ok = sym(D.h, "cuModuleLoadData", D.ModuleLoadData, D.why) && sym(D.h, "cuModuleGetFunction", D.ModuleGetFunction, D.why) && sym(D.h, "cuModuleUnload", D.ModuleUnload, D.why) &&
                  sym(D.h, "cuLaunchKernel", D.LaunchKernel, D.why) && sym(D.h, "cuFuncSetAttribute", D.FuncSetAttribute, D.why) &&
                  sym(D.h, "cuFuncGetAttribute", D.FuncGetAttribute, D.why) && sym(D.h, "cuGetErrorString", D.GetErrorString, D.why);
        if (!ok) { dlclose(D.h); D.h = nullptr; }
    });
    return &D;
}

// ------------------------------------------------------------------ per-robot cache of compiled programs
struct Program {
    bool ok = false;
    std::string why;          // why not, when !ok
    std::string cubin;        // sm_90a image
    std::vector<double> consts;
    int nin = 1, nout = 0, nout2 = 0, nres = 0, nc = 1, tpw = 1;
    int wpb = 4;    // warps per block
    int nblk = 0;   // derivative kernels: output blocks of n x n reals (2 or 3), each its own array
    const char *entry = "k_rne_spec";
    int n_mul = 0, n_fma = 0, n_add = 0, regs = 0;
    size_t smem = 0;
    std::map<int, CUfunction> fn; // per device
    std::vector<CUmodule> modules; // loaded images, unloaded with the robot handle
};
typedef std::tuple<int, int, int, int> Key; // mode, dtype, grav_mask, has_fext
struct SpecCache {
    std::mutex mu;
    std::map<Key, Program> progs;
    ~SpecCache();
};

SpecCache::~SpecCache()
{ // release the loaded images (best effort: the context may already be gone at interpreter shutdown)
    Driver *D = driver();
    if (!D->h) return;
    for (auto &kv : progs)
        for (CUmodule m : kv.second.modules) D->ModuleUnload(m);
}

int spec_setting()
{ // read at every call so a process can switch (tests run both paths)
    const char *e = getenv("B2K_RNE_SPEC");
    return e ? atoi(e) : 1;
}

int gcd_i(int a, int b) { return b ? gcd_i(b, a % b) : a; }

typedef std::function<int(b2k_gen_out &)> GenFn; // runs the code generator for one (robot, operation, pattern)

std::string build_source(const GenFn &gen, int n, int mode, int dtype, Program &p, std::vector<std::string> &defs, const char *kernel_text)
{
    b2k_gen_out g;
    if (gen(g)) { p.why = g.error; return std::string(); }
    p.consts = g.consts;
    p.nc = (int)g.consts.size();
    p.n_mul = g.n_mul; p.n_fma = g.n_fma; p.n_add = g.n_add;
    const b2k_rne_op_s &op = B2K_RNE_OPS[mode];
    p.nin = op.nin;
    // the rollout kernel (kRollout) runs the ACCEL / ACCEL_DERIV rows in its own 64-lane blocks: none of the tile sizing below
    const bool roll = kernel_text == kRollout;
    const bool deriv = !roll && (mode == B2K_GEN_RNE_DERIV || mode == B2K_GEN_ACCEL_DERIV), reg = mode == B2K_GEN_TREE_REGRESSOR;
    p.nout = op.out_row(0, n);
    p.nout2 = op.nout > 1 ? op.out_row(1, n) : 0; // tau (N, n) and the base wrench (N, 6)
    p.nres = mode == B2K_GEN_ACCEL ? n * n + n : p.nout + p.nout2;
    const int es = dtype == B2K_F64 ? 8 : 4;
    // one-row-per-lane reads of an exact-image tile: conflict degree gcd(row words, banks served per wavefront)
    const int padin = gcd_i(n * es / 4, es == 8 ? 32 : 32) > (es == 8 ? 4 : 2) ? 1 : 0;
    const int ldi = padin ? (n | 1) : n;
    const size_t in_bytes = ((size_t)32 * ldi * es + 15) & ~(size_t)15;
    // tiles per warp (double-buffered inputs when > 1).  fp64: no gain -- the kernel is bound by instruction issue (2-cycle
    // FP64 issue + integer / control), and the second buffer costs registers.  fp32: the whole recursion is ~480 issued
    // instructions per row, short enough for the tile-load latency to show (ncu: long-scoreboard the top stall), and two
    // tiles per warp with 8 resident blocks measured faster on the Puma.
    // Tried and dropped (commit b8738be): two fp32 rows per
    // lane as f32x2 pairs (FFMA2 / FMUL2: 35 % fewer issued instructions, same time -- an FFMA2 still holds the FP32
    // pipe for two cycles and the kernel is not bound by issue at this size) and a persistent grid-stride loop with
    // double-buffered tiles (fp32 equal, fp64 slower: the second buffer's registers spill).
    const bool light = mode == B2K_GEN_RNE || mode == B2K_GEN_GRAVLOAD || mode == B2K_GEN_ITORQUE || mode == B2K_GEN_RNE_WRENCH;
    const int tpw = (dtype == B2K_F32 && light) ? 2 : 1;
    p.tpw = tpw;
    p.smem = 4 * ((tpw > 1 ? 2 : 1) * p.nin * in_bytes + (size_t)32 * (p.nout + p.nout2) * es);
    if (deriv) { // one stage of 32 x n x n reals per output block and warp; as many warps per block as fit, up to 4
        p.nblk = op.nout;
        p.nout = n * n; p.nout2 = 0;
        p.nres = n * n + n;
        const size_t warp_bytes = p.nin * in_bytes + (size_t)p.nblk * 32 * n * n * es;
        p.wpb = (int)std::min<size_t>(4, (220 * 1024) / warp_bytes);
        p.smem = (size_t)std::max(p.wpb, 1) * warp_bytes;
    }
    if (reg) { // per warp the input tiles and the slab of one joint row (32 x 10 n reals, odd stride); up to 4 warps
        const size_t warp_bytes = p.nin * in_bytes + (((size_t)32 * ((10 * n) | 1) * es + 15) & ~(size_t)15);
        p.wpb = (int)std::min<size_t>(4, (220 * 1024) / warp_bytes);
        p.smem = (size_t)std::max(p.wpb, 1) * warp_bytes;
    }
    if (roll) { // static shared memory only (the slab of the sensitivities); SENS selects the program
        p.smem = 0; p.wpb = 2;
        defs.push_back(std::string("-DSENS=") + (mode == B2K_GEN_ACCEL_DERIV ? "1" : "0"));
    }
    if (p.smem > 220 * 1024) { p.why = "a tile of this operation does not fit the shared memory of an SM (" + std::to_string(p.smem) + " B)"; return std::string(); }
    int minb = (int)((200 * 1024) / (p.smem + 1024));
    // resident blocks to aim for (swept: fp64 96 registers / 5 blocks, fp32 64 registers / 8 blocks)
    const int want = deriv || reg ? 1 : light ? (es == 8 ? 5 : 8) : (es == 8 ? 2 : 3);
    if (minb > want) minb = want;
    if (minb < 1) minb = 1;
    auto D = [&](const char *k, long long v) { defs.push_back(std::string("-D") + k + "=" + std::to_string(v)); };
    defs.push_back(std::string("-DREAL=") + (es == 8 ? "double" : "float"));
    D("REAL_IS_F64", es == 8);
    D("NJ", n); D("NC", p.nc); D("MODE", mode); D("NIN", p.nin); D("NOUT", p.nout); D("NRES", p.nres); D("PADIN", padin); D("MINB", minb); D("TPW", tpw);
    if (p.nout2) D("NOUT2", p.nout2);
    if (deriv || reg) D("WPB", p.wpb);
    // in1 / in2 of the generated function are the second / third input rows; the RNE proper names them qd / qdd
    return std::string(kPrologue) + g.source + (kernel_text ? kernel_text : std::string(kTileIn) + (deriv ? kDeriv : reg ? kReg : kKernel));
}

void compile(const GenFn &gen, int n, const Key &key, Program &p)
{
    const int mode = std::get<0>(key) % 100, dtype = std::get<1>(key);
    Nvrtc *N = nvrtc();
    if (!N->h) { p.why = N->why; return; }
    std::vector<std::string> defs;
    const bool fdyn = std::get<0>(key) / 100 == 2, roll = std::get<0>(key) / 100 == 3;
    if (fdyn) p.entry = "k_fdyn";
    else if (roll) p.entry = "k_rollout";
    else if (mode == B2K_GEN_RNE_DERIV || mode == B2K_GEN_ACCEL_DERIV) p.entry = "k_rne_deriv_spec";
    else if (mode == B2K_GEN_TREE_REGRESSOR) p.entry = "k_rne_regressor_spec";
    const std::string src = build_source(gen, n, mode, dtype, p, defs, fdyn ? kFdyn : roll ? kRollout : nullptr);
    if (src.empty()) return;
    std::vector<std::string> opts = {"--gpu-architecture=sm_90a", "--std=c++17"};
    if (roll) opts.push_back("--fmad=false"); // no contraction: both rollout programs round the states alike
    if (getenv("B2K_RNE_SPEC_LINEINFO")) opts.push_back("-lineinfo");
    for (auto &d : defs) opts.push_back(d);
    std::vector<const char *> copts;
    for (auto &s : opts) copts.push_back(s.c_str());
    nvrtcProgram prog;
    nvrtcResult rc = N->CreateProgram(&prog, src.c_str(), "b2k_rne_spec.cu", 0, nullptr, nullptr);
    if (rc != NVRTC_SUCCESS) { p.why = std::string("nvrtcCreateProgram: ") + N->GetErrorString(rc); return; }
    rc = N->CompileProgram(prog, (int)copts.size(), copts.data());
    if (rc != NVRTC_SUCCESS) {
        size_t ls = 0;
        N->GetProgramLogSize(prog, &ls);
        std::string log(ls, '\0');
        if (ls) N->GetProgramLog(prog, &log[0]);
        p.why = std::string("nvrtcCompileProgram: ") + N->GetErrorString(rc) + "\n" + log.substr(0, 1500);
        N->DestroyProgram(&prog);
        return;
    }
    size_t cs = 0;
    N->GetCUBINSize(prog, &cs);
    p.cubin.assign(cs, '\0');
    N->GetCUBIN(prog, &p.cubin[0]);
    N->DestroyProgram(&prog);
    if (const char *dir = getenv("B2K_RNE_SPEC_DUMP")) { // for cuobjdump / offline inspection
        char name[512];
        snprintf(name, sizeof(name), "%s/rne_spec_m%d_%s_n%d_g%d_f%d", dir, std::get<0>(key), dtype == B2K_F64 ? "f64" : "f32", n, std::get<2>(key), std::get<3>(key));
        if (FILE *f = fopen((std::string(name) + ".cubin").c_str(), "wb")) { fwrite(p.cubin.data(), 1, p.cubin.size(), f); fclose(f); }
        if (FILE *f = fopen((std::string(name) + ".cu").c_str(), "w")) {
            for (auto &d : defs) fprintf(f, "// %s\n", d.c_str());
            fputs(src.c_str(), f);
            fclose(f);
        }
    }
    p.ok = true;
}

Program *get_program(SpecCache *c, const GenFn &gen, int n, const Key &key)
{
    if (!c) return nullptr;
    std::lock_guard<std::mutex> lk(c->mu);
    auto it = c->progs.find(key);
    if (it == c->progs.end()) {
        Program &p = c->progs[key];
        compile(gen, n, key, p);
        if (!p.ok && getenv("B2K_VERBOSE")) fprintf(stderr, "b2kin: RNE specialisation unavailable (%s); using the generic kernel\n", p.why.c_str());
        return &p;
    }
    return &it->second;
}

GenFn dh_gen(const b2k_rne_s *r, const Key &key)
{
    return [r, key](b2k_gen_out &g) {
        b2k_gen_opts o;
        o.mode = std::get<0>(key); o.grav_mask = std::get<2>(key); o.has_fext = std::get<3>(key);
        if (o.mode % 100 == B2K_GEN_ACCEL && r->mdh && (int)r->L[0][4] != 0) {
            // the prismatic-first-joint treatment kept for modified DH (ne.c:187-204) makes M non-symmetric, and the
            // accel kernels here solve with a pivot-free LDL^T that reads only M's lower triangle
            g.error = "accel of a modified-DH arm with a prismatic first joint needs the pivoted solve of the generic kernel";
            return -1;
        }
        return b2k_rne_generate(r, o, g);
    };
}

int get_function(Program *p, CUfunction *out)
{
    Driver *D = driver();
    if (!D->h) { p->ok = false; p->why = D->why; return -1; }
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return -1;
    auto it = p->fn.find(dev);
    if (it != p->fn.end()) { *out = it->second; return 0; }
    cudaFree(0); // make sure the runtime's primary context exists and is current on this thread
    CUmodule mod;
    CUresult rc = D->ModuleLoadData(&mod, p->cubin.data());
    const char *es = nullptr;
    if (rc != CUDA_SUCCESS) { D->GetErrorString(rc, &es); p->ok = false; p->why = std::string("cuModuleLoadData: ") + (es ? es : "?"); return -1; }
    CUfunction fn;
    rc = D->ModuleGetFunction(&fn, mod, p->entry);
    if (rc != CUDA_SUCCESS) { D->GetErrorString(rc, &es); p->ok = false; p->why = std::string("cuModuleGetFunction: ") + (es ? es : "?"); return -1; }
    if (p->smem > 48 * 1024) {
        rc = D->FuncSetAttribute(fn, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)p->smem);
        if (rc != CUDA_SUCCESS) { D->GetErrorString(rc, &es); p->ok = false; p->why = std::string("cuFuncSetAttribute: ") + (es ? es : "?"); return -1; }
    }
    D->FuncGetAttribute(&p->regs, CU_FUNC_ATTRIBUTE_NUM_REGS, fn);
    p->fn[dev] = fn;
    p->modules.push_back(mod);
    *out = fn;
    return 0;
}

template <typename real>
struct SpecParams { // byte image of the kernel's SpecP for NC constants (built in a buffer)
};

// Builds the kernel's parameter block SpecP { real C[NC]; real grav[3]; real fext[6]; real offset[NJ]; TrigC trig; } and
// launches `ntiles` full tiles on `st`.
std::vector<unsigned char> spec_params(Program *p, int n, int dtype, const double *offset, const double *grav, const double *fext)
{
    const int es = dtype == B2K_F64 ? 8 : 4;
    const int nreal = p->nc + 3 + 6 + n + 18;
    std::vector<unsigned char> pb((size_t)nreal * es);
    auto put = [&](int idx, double v) {
        if (es == 8) memcpy(&pb[(size_t)idx * 8], &v, 8);
        else { float f = (float)v; memcpy(&pb[(size_t)idx * 4], &f, 4); }
    };
    int o = 0;
    for (int k = 0; k < p->nc; k++) put(o++, p->consts[k]);
    for (int k = 0; k < 3; k++) put(o++, grav ? grav[k] : 0.0);
    for (int k = 0; k < 6; k++) put(o++, fext ? fext[k] : 0.0);
    for (int j = 0; j < n; j++) put(o++, offset ? offset[j] : 0.0);
    if (es == 8) {
        TrigC<double> t;
        b2k_fill_trig<double>(t);
        memcpy(&pb[(size_t)o * 8], &t, sizeof(t));
    } else {
        TrigC<float> t;
        b2k_fill_trig<float>(t);
        memcpy(&pb[(size_t)o * 4], &t, sizeof(t));
    }
    return pb;
}

int launch_tiles(Program *p, CUfunction fn, int n, int dtype, const double *offset, const void *in0, const void *in1, const void *in2,
                 void *out, void *out2, long long ntiles, const double *grav, const double *fext, cudaStream_t st, void *out3 = nullptr)
{
    std::vector<unsigned char> pb = spec_params(p, n, dtype, offset, grav, fext);
    long long nt = ntiles;
    void *args[8] = {pb.data(), (void *)&in0, (void *)&in1, (void *)&in2, (void *)&out, (void *)&nt, nullptr, nullptr};
    if (p->nblk) { args[5] = (void *)&out2; args[6] = (void *)&out3; args[7] = (void *)&nt; } // k_rne_deriv_spec(..., out0, out1, out2, ntiles)
    else if (p->nout2) { args[5] = (void *)&out2; args[6] = (void *)&nt; } // k_rne_spec(..., out, out2, ntiles)
    const long long per_block = (long long)p->wpb * p->tpw;
    const unsigned grid = (unsigned)((ntiles + per_block - 1) / per_block);
    CUresult rc = driver()->LaunchKernel(fn, grid, 1, 1, 32 * p->wpb, 1, 1, (unsigned)p->smem, (CUstream)st, args, nullptr);
    if (rc != CUDA_SUCCESS) {
        const char *es2 = nullptr;
        driver()->GetErrorString(rc, &es2);
        b2k_set_error("cuLaunchKernel(k_rne_spec): %s", es2 ? es2 : "?");
        return B2K_ERR_CUDA;
    }
    b2k_count_launch();
    return B2K_OK;
}

int grav_mask_of(const double *g)
{
    int m = 0;
    if (g)
        for (int k = 0; k < 3; k++)
            if (g[k] != 0.0) m |= 1 << k;
    return m;
}

} // namespace

void b2k_rne_spec_attach(b2k_rne_s *r) { r->spec = new SpecCache(); }
void b2k_rne_spec_detach(b2k_rne_s *r)
{
    delete static_cast<SpecCache *>(r->spec);
    r->spec = nullptr;
}

// Tries the specialised kernel for the first (N / 32) * 32 rows.  Returns the number of rows it served (0 when the
// call must go to the generic kernel entirely), or a negative b2k_status when B2K_RNE_SPEC=2 demands it and it failed.
long long b2k_rne_spec_launch(const b2k_rne_s *r, int mode, int dtype, const void *in0, const void *in1, const void *in2,
                              long long nrows, const double *grav, const double *fext, void *out, void *out2, cudaStream_t st)
{
    const int setting = spec_setting();
    if (setting == 0 || !r->spec) return 0;
    auto refuse = [&](const std::string &why) -> long long {
        if (setting == 2) { b2k_set_error("RNE specialisation required (B2K_RNE_SPEC=2) but unavailable: %s", why.c_str()); return B2K_ERR_INVALID; }
        return 0;
    };
    const long long ntiles = nrows / 32;
    if (ntiles == 0) return 0;
    const uintptr_t al = (uintptr_t)in0 | (uintptr_t)(in1 ? in1 : in0) | (uintptr_t)(in2 ? in2 : in0) | (uintptr_t)out | (uintptr_t)(out2 ? out2 : out);
    if (al & 15) return refuse("arrays are not 16-byte aligned");
    const bool rne = mode == B2K_GEN_RNE || mode == B2K_GEN_RNE_WRENCH;
    int has_fext = 0;
    if (rne && fext)
        for (int k = 0; k < 6; k++) has_fext |= (fext[k] != 0.0);
    const bool uses_grav = B2K_RNE_OPS[mode].grav;
    const Key key(mode, dtype, uses_grav ? grav_mask_of(grav) : 0, has_fext);
    Program *p = get_program(static_cast<SpecCache *>(r->spec), dh_gen(r, key), r->n, key);
    if (!p || !p->ok) return refuse(p ? p->why : "no cache");
    CUfunction fn;
    {
        SpecCache *c = static_cast<SpecCache *>(r->spec);
        std::lock_guard<std::mutex> lk(c->mu);
        if (get_function(p, &fn)) return refuse(p->why);
    }
    double offset[B2K_MAX_JOINTS];
    for (int j = 0; j < r->n; j++) offset[j] = r->L[j][5];
    const int lrc = launch_tiles(p, fn, r->n, dtype, offset, in0, in1, in2, out, out2, ntiles, uses_grav ? grav : nullptr,
                                 has_fext ? fext : nullptr, st);
    if (lrc) return lrc;
    return ntiles * 32;
}

// ------------------------------------------------------------------ C ABI: introspection (tests, bench, DESIGN numbers)
extern "C" int b2k_rne_codegen(b2k_rne_t r, int mode, int grav_mask, int has_fext, char *src, int64_t src_cap, double *consts,
                               int32_t consts_cap, int32_t *n_consts, int32_t *counts)
{
    if (!r) { b2k_set_error("b2k_rne_codegen: rne handle is NULL"); return B2K_ERR_INVALID; }
    b2k_gen_opts o;
    o.mode = mode; o.grav_mask = grav_mask; o.has_fext = has_fext;
    b2k_gen_out g;
    if (b2k_rne_generate(r, o, g)) { b2k_set_error("b2k_rne_codegen: %s", g.error.c_str()); return B2K_ERR_INVALID; }
    if (n_consts) *n_consts = (int32_t)g.consts.size();
    if (counts) { counts[0] = g.n_mul; counts[1] = g.n_fma; counts[2] = g.n_add; }
    if (src) {
        if ((int64_t)g.source.size() + 1 > src_cap) { b2k_set_error("b2k_rne_codegen: source needs %zu bytes", g.source.size() + 1); return B2K_ERR_INVALID; }
        memcpy(src, g.source.c_str(), g.source.size() + 1);
    }
    if (consts) {
        if ((int32_t)g.consts.size() > consts_cap) { b2k_set_error("b2k_rne_codegen: %zu constants", g.consts.size()); return B2K_ERR_INVALID; }
        memcpy(consts, g.consts.data(), g.consts.size() * sizeof(double));
    }
    return B2K_OK;
}

extern "C" int b2k_rne_spec_info(b2k_rne_t r, int mode, int dtype, const double *grav, int has_fext, char *buf, int64_t cap)
{
    if (!r || !buf || cap < 1) { b2k_set_error("b2k_rne_spec_info: bad arguments"); return B2K_ERR_INVALID; }
    std::string s;
    if (spec_setting() == 0) s = "generic (B2K_RNE_SPEC=0)";
    else {
        {
            // mode 200 + m: the forward-dynamics integrator built around operation m (only m = accel exists)
            const int gm = mode % 100;
            const bool ug = gm >= 0 && gm < B2K_GEN_NOPS && B2K_RNE_OPS[gm].grav;
            const Key key(mode, dtype, ug ? grav_mask_of(grav) : 0, has_fext);
            const Key gkey(gm, dtype, ug ? grav_mask_of(grav) : 0, has_fext);
            // b2k_rne_derivatives / b2k_rne_accel_derivatives run the generic kernel; their generated rows serve rollouts only
            const bool generic = mode == B2K_GEN_RNE_DERIV || mode == B2K_GEN_ACCEL_DERIV;
            Program *p = generic ? nullptr : get_program(static_cast<SpecCache *>(r->spec), dh_gen(r, gkey), r->n, key);
            if (generic) s = "generic (the derivatives of DH arms are served by the generic kernel)";
            else if (!p || !p->ok) s = std::string("generic (") + (p ? p->why : "no cache") + ")";
            else {
                char t[256];
                snprintf(t, sizeof(t), "%s<%s,n=%d,mode=%d>: %d mul + %d fma + %d add per row, %d constants, %d regs, %zu B smem/block, %d tiles/warp",
                         p->entry, dtype == B2K_F64 ? "double" : "float", r->n, mode, p->n_mul, p->n_fma, p->n_add, p->nc, p->regs, p->smem, p->tpw);
                s = t;
            }
        }
    }
    snprintf(buf, (size_t)cap, "%s", s.c_str());
    return B2K_OK;
}

// ------------------------------------------------------------------ rigid-body trees: Robot.rne (reference Robot.py:1704-1903)
// There is no pre-compiled kernel for an arbitrary tree: the recursion is always generated for the robot at hand
// (b2k_tree_generate) and compiled with NVRTC at first use; without NVRTC / the driver API the call fails with an error.
extern "C" int b2k_tree_create(int n, const int32_t *parent, const int32_t *axis, const int32_t *flip, const int32_t *jindex,
                               const double *C, const double *I6, b2k_tree_t *out)
{
    const char *fn = "b2k_tree_create";
    if (!out) { b2k_set_error("%s: out is NULL", fn); return B2K_ERR_INVALID; }
    *out = nullptr;
    if (n < 1 || n > B2K_TREE_MAX || !parent || !axis || !flip || !jindex || !C || !I6) {
        b2k_set_error("%s: n = %d outside 1..%d or a NULL table", fn, n, B2K_TREE_MAX);
        return B2K_ERR_INVALID;
    }
    bool seen[B2K_TREE_MAX] = {false};
    for (int j = 0; j < n; j++) {
        if (parent[j] < -1 || parent[j] >= j) { b2k_set_error("%s: parent[%d] = %d must precede the group (or be -1)", fn, j, parent[j]); return B2K_ERR_INVALID; }
        if (axis[j] < 0 || axis[j] > 5) { b2k_set_error("%s: axis[%d] = %d is not B2K_RX..B2K_TZ", fn, j, axis[j]); return B2K_ERR_INVALID; }
        if (jindex[j] < 0 || jindex[j] >= n || seen[jindex[j]]) { b2k_set_error("%s: the jindices must be a permutation of 0..n-1", fn); return B2K_ERR_INVALID; }
        seen[jindex[j]] = true;
    }
    b2k_tree_s *t = (b2k_tree_s *)calloc(1, sizeof(b2k_tree_s));
    if (!t) { b2k_set_error("%s: out of memory", fn); return B2K_ERR_ALLOC; }
    t->n = n;
    for (int j = 0; j < n; j++) {
        t->parent[j] = parent[j]; t->axis[j] = axis[j]; t->flip[j] = flip[j] ? 1 : 0; t->jindex[j] = jindex[j];
        memcpy(t->C[j], C + 12 * j, 12 * sizeof(double));
        memcpy(t->I6[j], I6 + 36 * j, 36 * sizeof(double));
    }
    t->spec = new SpecCache();
    *out = t;
    return B2K_OK;
}

extern "C" int b2k_tree_destroy(b2k_tree_t t)
{
    if (t) delete static_cast<SpecCache *>(t->spec);
    free(t);
    return B2K_OK;
}

static GenFn tree_gen(b2k_tree_t t, int mode, int gmask)
{
    return [t, mode, gmask](b2k_gen_out &g) {
        b2k_gen_opts o;
        o.mode = mode; o.grav_mask = gmask; o.has_fext = 0;
        return b2k_tree_generate(t, o, g);
    };
}

static Program *tree_program(b2k_tree_t t, int mode, int dtype, int gmask)
{
    return get_program(static_cast<SpecCache *>(t->spec), tree_gen(t, mode, gmask), t->n, Key(100 + mode, dtype, gmask, 0));
}

// Robot.rne (mode 0), the operations DynamicsMixin builds on it (modes 1-5: inertia, gravload, itorque, coriolis, accel),
// their derivatives (modes 7, 8; TREE_DERIVS: the b2k_tree_derivatives entry point) and the regressor (mode 10,
// TREE_REGRESSOR) for a rigid-body tree: the generated kernel on the full tiles, one padded tile for the ragged tail.
// out[0..nout) are the operation's output arrays.
enum TreeEntry { TREE_DYN, TREE_DERIVS, TREE_REGRESSOR };
static int tree_run(const char *fn, b2k_tree_t t, int mode, TreeEntry entry, int dtype, const void *in0, const void *in1,
                    const void *in2, int64_t N, const double *grav, void *const out[3], void *stream)
{
    if (!t) { b2k_set_error("%s: tree handle is NULL", fn); return B2K_ERR_INVALID; }
    const bool derivs = entry == TREE_DERIVS;
    if (entry == TREE_REGRESSOR ? mode != B2K_GEN_TREE_REGRESSOR
        : derivs                ? (mode != B2K_GEN_RNE_DERIV && mode != B2K_GEN_ACCEL_DERIV)
                                : (mode < B2K_GEN_RNE || mode > B2K_GEN_ACCEL)) {
        if (derivs) b2k_set_error("%s: operation %d is not B2K_DYN_RNE_DERIV or B2K_DYN_ACCEL_DERIV", fn, mode);
        else b2k_set_error("%s: operation %d is not one of B2K_DYN_*", fn, mode);
        return B2K_ERR_INVALID;
    }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    const b2k_rne_op_s &op = B2K_RNE_OPS[mode];
    const int nin = op.nin, nout = op.nout;
    bool missing = false;
    for (int o = 0; o < nout; o++) missing |= !out[o];
    if (N < 0 || (N > 0 && (!in0 || (nin >= 2 && !in1) || (nin >= 3 && !in2) || missing))) { b2k_set_error("%s: bad arguments", fn); return B2K_ERR_INVALID; }
    for (int o = nout; o < 3; o++)
        if (out[o]) { b2k_set_error("%s: operation %d has %d outputs: %s must be NULL", fn, mode, nout, o == 2 ? "out2" : "out1"); return B2K_ERR_INVALID; }
    const bool ug = op.grav;
    if (ug && !grav) { b2k_set_error("%s: grav is NULL (pass MINUS the robot's gravity: a_grav of Robot.rne)", fn); return B2K_ERR_INVALID; }
    uintptr_t al = (uintptr_t)in0 | (uintptr_t)(nin >= 2 ? in1 : in0) | (uintptr_t)(nin >= 3 ? in2 : in0);
    for (int o = 0; o < nout; o++) al |= (uintptr_t)out[o];
    if (al & 15) { b2k_set_error("%s: arrays must be 16-byte aligned", fn); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(in0);
    Program *p = tree_program(t, mode, dtype, ug ? grav_mask_of(grav) : 0);
    if (!p || !p->ok) {
        b2k_set_error("%s: the kernel for this robot could not be built (%s); Robot.rne has no pre-compiled kernel", fn, p ? p->why.c_str() : "no cache");
        return B2K_ERR_INVALID;
    }
    CUfunction f;
    {
        SpecCache *c = static_cast<SpecCache *>(t->spec);
        std::lock_guard<std::mutex> lk(c->mu);
        if (get_function(p, &f)) { b2k_set_error("%s: %s", fn, p->why.c_str()); return B2K_ERR_CUDA; }
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int n = t->n;
    const size_t es = dtype == B2K_F64 ? 8 : 4, rowb = (size_t)n * es, orowb = (size_t)p->nout * es;
    const long long ntiles = N / 32, tail = N - ntiles * 32;
    const double *gv = ug ? grav : nullptr;
    int rc = B2K_OK;
    if (ntiles) rc = launch_tiles(p, f, n, dtype, nullptr, in0, in1, in2, out[0], out[1], ntiles, gv, nullptr, st, out[2]);
    if (rc == B2K_OK && tail) { // ragged tail: one padded tile through stream-ordered scratch
        b2k_keep_mempool();
        char *scr = nullptr;
        B2K_CUDA(cudaMallocAsync((void **)&scr, 3 * 32 * rowb + nout * 32 * orowb, st));
        cudaMemsetAsync(scr, 0, 3 * 32 * rowb, st);
        const size_t off = (size_t)ntiles * 32 * rowb;
        const void *src[3] = {in0, in1, in2};
        for (int i = 0; i < nin; i++) cudaMemcpyAsync(scr + i * 32 * rowb, (const char *)src[i] + off, tail * rowb, cudaMemcpyDeviceToDevice, st);
        char *so[3] = {nullptr, nullptr, nullptr};
        for (int o = 0; o < nout; o++) so[o] = scr + 3 * 32 * rowb + o * 32 * orowb;
        rc = launch_tiles(p, f, n, dtype, nullptr, scr, scr + 32 * rowb, scr + 2 * 32 * rowb, so[0], so[1], 1, gv, nullptr, st, so[2]);
        for (int o = 0; o < nout; o++)
            cudaMemcpyAsync((char *)out[o] + (size_t)ntiles * 32 * orowb, so[o], tail * orowb, cudaMemcpyDeviceToDevice, st);
        cudaFreeAsync(scr, st);
        cudaError_t e = cudaGetLastError();
        if (rc == B2K_OK && e != cudaSuccess) rc = b2k_cuda_fail(e, "tail tile of a tree kernel");
    }
    return rc;
}

extern "C" int b2k_tree_rne(b2k_tree_t t, int dtype, const void *q, const void *qd, const void *qdd, int64_t N, const double *grav,
                            void *tau, void *stream)
{
    void *const out[3] = {tau, nullptr, nullptr};
    return tree_run("b2k_tree_rne", t, B2K_GEN_RNE, TREE_DYN, dtype, q, qd, qdd, N, grav, out, stream);
}

extern "C" int b2k_tree_dyn(b2k_tree_t t, int op, int dtype, const void *in0, const void *in1, const void *in2, int64_t N,
                            const double *grav, void *out, void *stream)
{
    void *const outs[3] = {out, nullptr, nullptr};
    return tree_run("b2k_tree_dyn", t, op, TREE_DYN, dtype, in0, in1, in2, N, grav, outs, stream);
}

extern "C" int b2k_tree_derivatives(b2k_tree_t t, int op, int dtype, const void *q, const void *qd, const void *x, int64_t N,
                                    const double *grav, void *out0, void *out1, void *out2, void *stream)
{
    void *const outs[3] = {out0, out1, out2};
    return tree_run("b2k_tree_derivatives", t, op, TREE_DERIVS, dtype, q, qd, x, N, grav, outs, stream);
}

extern "C" int b2k_tree_regressor(b2k_tree_t t, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                                  const double *grav, void *Y, void *stream)
{
    void *const outs[3] = {Y, nullptr, nullptr};
    return tree_run("b2k_tree_regressor", t, B2K_GEN_TREE_REGRESSOR, TREE_REGRESSOR, dtype, q, qd, qdd, N, grav, outs, stream);
}

int b2k_tree_regressor_rows(b2k_tree_t t, int dtype, const b2k_rne_args &a, cudaStream_t st)
{
    void *const outs[3] = {a.out[0], nullptr, nullptr};
    return tree_run("b2k_tree_regressor_gram", t, B2K_GEN_TREE_REGRESSOR, TREE_REGRESSOR, dtype, a.in[0], a.in[1], a.in[2],
                    a.nrows, a.grav, outs, st);
}

int b2k_tree_regressor_gram_f32(b2k_tree_t, int, const b2k_rne_args &, const void *, const double *, double *, double *, double *,
                                cudaStream_t);
int b2k_tree_regressor_gram_f64(b2k_tree_t, int, const b2k_rne_args &, const void *, const double *, double *, double *, double *,
                                cudaStream_t);

// The normal equations of the tree regressor (b2k_rne.cuh: regressor_gram, shared with the DH arms).  Every argument is
// checked, and the kernel built, before any CUDA call.
extern "C" int b2k_tree_regressor_gram(b2k_tree_t t, int dtype, const void *q, const void *qd, const void *qdd, const void *tau,
                                       int64_t N, const double *grav, const double *weights, double *G, double *b, double *s,
                                       void *stream)
{
    const char *fn = "b2k_tree_regressor_gram";
    if (!t) { b2k_set_error("%s: tree handle is NULL", fn); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: N is negative", fn); return B2K_ERR_INVALID; }
    if (!grav) { b2k_set_error("%s: grav is NULL (pass MINUS the robot's gravity: a_grav of Robot.rne)", fn); return B2K_ERR_INVALID; }
    const int es = dtype == B2K_F64 ? 8 : 4, n = t->n;
    int rc;
    const char *names[3] = {"q", "qd", "qdd"};
    const void *ins[3] = {q, qd, qdd};
    for (int i = 0; i < 3; i++)
        if ((rc = b2k_check_array(fn, names[i], ins[i], N, 16))) return rc;
    if ((rc = b2k_check_array(fn, "tau", tau, N, es))) return rc;
    if (weights)
        for (int j = 0; j < n; j++)
            if (!isfinite(weights[j]) || weights[j] < 0) {
                b2k_set_error("%s: weights[%d] = %g is not a finite value >= 0", fn, j, weights[j]);
                return B2K_ERR_INVALID;
            }
    // the sums are written whatever N is (zeros for N = 0)
    if ((rc = b2k_check_array(fn, "G", G, 1, 8)) || (rc = b2k_check_array(fn, "b", b, 1, 8)) || (rc = b2k_check_array(fn, "s", s, 1, 8)))
        return rc;
    const b2k_rne_args a = {{q, qd, qdd}, {nullptr}, N, grav, nullptr};
    if (N > 0) { // the generated kernel is built before any CUDA call, so that a tree it cannot serve leaves no work queued
        Program *p = tree_program(t, B2K_GEN_TREE_REGRESSOR, dtype, grav_mask_of(grav));
        if (!p || !p->ok) {
            b2k_set_error("%s: the kernel for this robot could not be built (%s)", fn, p ? p->why.c_str() : "no cache");
            return B2K_ERR_INVALID;
        }
    }
    B2K_ON_DEVICE_OF(G);
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) {
        const size_t p = 10 * (size_t)n;
        B2K_CUDA(cudaMemsetAsync(G, 0, p * p * sizeof(double), st));
        B2K_CUDA(cudaMemsetAsync(b, 0, p * sizeof(double), st));
        B2K_CUDA(cudaMemsetAsync(s, 0, sizeof(double), st));
        return B2K_OK;
    }
    return dtype == B2K_F64 ? b2k_tree_regressor_gram_f64(t, n, a, tau, weights, G, b, s, st)
                            : b2k_tree_regressor_gram_f32(t, n, a, tau, weights, G, b, s, st);
}

extern "C" int b2k_tree_codegen(b2k_tree_t t, int op, int grav_mask, char *src, int64_t src_cap, double *consts, int32_t consts_cap,
                                int32_t *n_consts, int32_t *counts)
{
    if (!t) { b2k_set_error("b2k_tree_codegen: tree handle is NULL"); return B2K_ERR_INVALID; }
    b2k_gen_out g;
    b2k_gen_opts o;
    o.mode = op; o.grav_mask = grav_mask; o.has_fext = 0;
    if (b2k_tree_generate(t, o, g)) { b2k_set_error("b2k_tree_codegen: %s", g.error.c_str()); return B2K_ERR_INVALID; }
    if (n_consts) *n_consts = (int32_t)g.consts.size();
    if (counts) { counts[0] = g.n_mul; counts[1] = g.n_fma; counts[2] = g.n_add; }
    if (src) {
        if ((int64_t)g.source.size() + 1 > src_cap) { b2k_set_error("b2k_tree_codegen: source needs %zu bytes", g.source.size() + 1); return B2K_ERR_INVALID; }
        memcpy(src, g.source.c_str(), g.source.size() + 1);
    }
    if (consts) {
        if ((int32_t)g.consts.size() > consts_cap) { b2k_set_error("b2k_tree_codegen: %zu constants", g.consts.size()); return B2K_ERR_INVALID; }
        memcpy(consts, g.consts.data(), g.consts.size() * sizeof(double));
    }
    return B2K_OK;
}

extern "C" int b2k_tree_info(b2k_tree_t t, int op, int dtype, const double *grav, char *buf, int64_t cap)
{
    if (!t || !buf || cap < 1) { b2k_set_error("b2k_tree_info: bad arguments"); return B2K_ERR_INVALID; }
    if (op == 300 + B2K_GEN_ACCEL || op == 300 + B2K_GEN_ACCEL_DERIV) { // the rollout kernels (b2k_tree_rollout)
        const int gm = grav_mask_of(grav);
        Program *p = get_program(static_cast<SpecCache *>(t->spec), tree_gen(t, op - 300, gm), t->n, Key(op, dtype, gm, 0));
        if (!p || !p->ok) snprintf(buf, (size_t)cap, "unavailable (%s)", p ? p->why.c_str() : "no cache");
        else
            snprintf(buf, (size_t)cap, "k_rollout<%s,tree n=%d,mode=%d>: %d mul + %d fma + %d add per stage, %d constants, %d regs",
                     dtype == B2K_F64 ? "double" : "float", t->n, op, p->n_mul, p->n_fma, p->n_add, p->nc, p->regs);
        return B2K_OK;
    }
    if (op < B2K_GEN_RNE || (op > B2K_GEN_ACCEL_DERIV && op != B2K_GEN_TREE_REGRESSOR) || op == B2K_GEN_RNE_WRENCH) {
        b2k_set_error("b2k_tree_info: operation %d is not one of B2K_DYN_*", op);
        return B2K_ERR_INVALID;
    }
    Program *p = tree_program(t, op, dtype, B2K_RNE_OPS[op].grav ? grav_mask_of(grav) : 0);
    if (!p || !p->ok) snprintf(buf, (size_t)cap, "unavailable (%s)", p ? p->why.c_str() : "no cache");
    else if (op == B2K_GEN_RNE)
        snprintf(buf, (size_t)cap, "k_rne_spec<%s,tree n=%d>: %d mul + %d fma + %d add per row, %d constants, %d regs, %zu B smem/block",
                 dtype == B2K_F64 ? "double" : "float", t->n, p->n_mul, p->n_fma, p->n_add, p->nc, p->regs, p->smem);
    else if (p->nblk || op == B2K_GEN_TREE_REGRESSOR)
        snprintf(buf, (size_t)cap, "%s<%s,tree n=%d,mode=%d>: %d mul + %d fma + %d add per row, %d constants, %d regs, %zu B smem/block, "
                 "%d warps/block",
                 p->entry, dtype == B2K_F64 ? "double" : "float", t->n, op, p->n_mul, p->n_fma, p->n_add, p->nc, p->regs, p->smem, p->wpb);
    else
        snprintf(buf, (size_t)cap, "k_rne_spec<%s,tree n=%d,mode=%d>: %d mul + %d fma + %d add per row, %d constants, %d regs, %zu B smem/block",
                 dtype == B2K_F64 ? "double" : "float", t->n, op, p->n_mul, p->n_fma, p->n_add, p->nc, p->regs, p->smem);
    return B2K_OK;
}


// ------------------------------------------------------------------ C ABI: forward-dynamics ensemble integrator
static int fdyn_run(const char *fn, SpecCache *cache, const GenFn &gen, int n, const double *offset, int dtype, const void *q0, const void *qd0, int64_t ntraj, double T, const double *grav,
                            int torque_mode, const double *tau, const void *tau_rows, const double *kp, const double *kd,
                            const double *qstar, double rtol, double atol, double max_step, double first_step, double dt, int grid,
                            int M, void *out_t, void *out_q, void *out_qd, int32_t *out_count, int32_t *out_status, void *stream)
{
    if (!cache) { b2k_set_error("%s: robot handle is NULL", fn); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (ntraj < 0 || (ntraj > 0 && (!q0 || !out_t || !out_q || !out_qd || !out_count || !out_status))) { b2k_set_error("%s: bad arguments", fn); return B2K_ERR_INVALID; }
    if (!(T > 0) || !(rtol > 0) || !(atol >= 0) || !(max_step > 0) || M < 1) { b2k_set_error("%s: T, rtol, max_step must be positive, atol non-negative, M >= 1", fn); return B2K_ERR_INVALID; }
    if (grid && !(dt > 0)) { b2k_set_error("%s: dt must be positive for a uniform output grid", fn); return B2K_ERR_INVALID; }
    if (!grav) { b2k_set_error("%s: grav is NULL (pass -robot.gravity like DHRobot.rne)", fn); return B2K_ERR_INVALID; }
    if (torque_mode < 0 || torque_mode > 3 || (torque_mode == 1 && !tau) || (torque_mode == 2 && !tau_rows) || (torque_mode == 3 && (!kp || !kd || !qstar))) {
        b2k_set_error("%s: torque_mode 0 none, 1 constant (tau), 2 per-trajectory (tau_rows), 3 PD (kp, kd, qstar)", fn);
        return B2K_ERR_INVALID;
    }
    if (ntraj == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(q0);
    const Key key(200 + B2K_GEN_ACCEL, dtype, grav_mask_of(grav), 0);
    Program *p = get_program(cache, gen, n, key);
    if (!p || !p->ok) { b2k_set_error("%s: the integrator kernel could not be built (%s)", fn, p ? p->why.c_str() : "no cache"); return B2K_ERR_INVALID; }
    CUfunction f;
    {
        std::lock_guard<std::mutex> lk(cache->mu);
        if (get_function(p, &f)) { b2k_set_error("%s: %s", fn, p->why.c_str()); return B2K_ERR_CUDA; }
    }
    const int es = dtype == B2K_F64 ? 8 : 4;
    std::vector<unsigned char> pb = spec_params(p, n, dtype, offset, grav, nullptr);
    // FdynP { real T, rtol, atol, max_step, first_step, dt; real kp[NJ], kd[NJ], qstar[NJ], tau[NJ]; int torque_mode, grid, M; }
    const int nreal = 6 + 4 * n;
    size_t fbytes = (size_t)nreal * es + 3 * sizeof(int);
    fbytes = (fbytes + es - 1) / es * es;
    std::vector<unsigned char> fb(fbytes, 0);
    auto put = [&](int idx, double v) {
        if (es == 8) memcpy(&fb[(size_t)idx * 8], &v, 8);
        else { float x = (float)v; memcpy(&fb[(size_t)idx * 4], &x, 4); }
    };
    const double head[6] = {T, rtol, atol, max_step, first_step, dt};
    for (int k = 0; k < 6; k++) put(k, head[k]);
    for (int j = 0; j < n; j++) {
        put(6 + j, kp ? kp[j] : 0.0); put(6 + n + j, kd ? kd[j] : 0.0); put(6 + 2 * n + j, qstar ? qstar[j] : 0.0); put(6 + 3 * n + j, tau ? tau[j] : 0.0);
    }
    const int tail[3] = {torque_mode, grid ? 1 : 0, M};
    memcpy(&fb[(size_t)nreal * es], tail, sizeof(tail));
    long long nt = ntraj;
    void *args[11] = {pb.data(), fb.data(), (void *)&q0, (void *)&qd0, (void *)&tau_rows, (void *)&out_t, (void *)&out_q, (void *)&out_qd,
                      (void *)&out_count, (void *)&out_status, (void *)&nt};
    const unsigned grid_dim = (unsigned)((ntraj + 63) / 64);
    CUresult rc = driver()->LaunchKernel(f, grid_dim, 1, 1, 64, 1, 1, 0, (CUstream)stream, args, nullptr);
    if (rc != CUDA_SUCCESS) {
        const char *es2 = nullptr;
        driver()->GetErrorString(rc, &es2);
        b2k_set_error("cuLaunchKernel(k_fdyn): %s", es2 ? es2 : "?");
        return B2K_ERR_CUDA;
    }
    b2k_count_launch();
    return B2K_OK;
}

extern "C" int b2k_rne_fdyn(b2k_rne_t r, int dtype, const void *q0, const void *qd0, int64_t ntraj, double T, const double *grav,
                            int torque_mode, const double *tau, const void *tau_rows, const double *kp, const double *kd,
                            const double *qstar, double rtol, double atol, double max_step, double first_step, double dt, int grid,
                            int M, void *out_t, void *out_q, void *out_qd, int32_t *out_count, int32_t *out_status, void *stream)
{
    if (!r) { b2k_set_error("b2k_rne_fdyn: rne handle is NULL"); return B2K_ERR_INVALID; }
    double offset[B2K_MAX_JOINTS];
    for (int j = 0; j < r->n; j++) offset[j] = r->L[j][5];
    const Key gkey(B2K_GEN_ACCEL, dtype, grav_mask_of(grav), 0);
    return fdyn_run("b2k_rne_fdyn", static_cast<SpecCache *>(r->spec), dh_gen(r, gkey), r->n, offset, dtype, q0, qd0, ntraj, T, grav,
                    torque_mode, tau, tau_rows, kp, kd, qstar, rtol, atol, max_step, first_step, dt, grid, M, out_t, out_q, out_qd,
                    out_count, out_status, stream);
}

// The same integrator around the accel recursion of a rigid-body tree (Robot.fdyn: DynamicsMixin.fdyn calls self.accel,
// which for a tree robot is n + 1 Python Robot.rne loops per stage in the reference).
extern "C" int b2k_tree_fdyn(b2k_tree_t t, int dtype, const void *q0, const void *qd0, int64_t ntraj, double T, const double *grav,
                             int torque_mode, const double *tau, const void *tau_rows, const double *kp, const double *kd,
                             const double *qstar, double rtol, double atol, double max_step, double first_step, double dt, int grid,
                             int M, void *out_t, void *out_q, void *out_qd, int32_t *out_count, int32_t *out_status, void *stream)
{
    if (!t) { b2k_set_error("b2k_tree_fdyn: tree handle is NULL"); return B2K_ERR_INVALID; }
    const int gmask = grav_mask_of(grav);
    GenFn gen = [t, gmask](b2k_gen_out &g) {
        b2k_gen_opts o;
        o.mode = B2K_GEN_ACCEL; o.grav_mask = gmask; o.has_fext = 0;
        return b2k_tree_generate(t, o, g);
    };
    return fdyn_run("b2k_tree_fdyn", static_cast<SpecCache *>(t->spec), gen, t->n, nullptr, dtype, q0, qd0, ntraj, T, grav, torque_mode,
                    tau, tau_rows, kp, kd, qstar, rtol, atol, max_step, first_step, dt, grid, M, out_t, out_q, out_qd, out_count,
                    out_status, stream);
}

// ------------------------------------------------------------------ C ABI: fixed-step rollouts with sensitivities
// gen(mode) runs the code generator of the robot for B2K_GEN_ACCEL (states only) or B2K_GEN_ACCEL_DERIV (sensitivities).
static int rollout_run(const char *fn, SpecCache *cache, const std::function<GenFn(int)> &gen, int n, const double *offset,
                       int dtype, const void *q0, const void *qd0, int64_t N, int32_t K, double dt, const double *grav,
                       const void *tau, int64_t tau_stride, void *q, void *qd, void *A, void *B, void *stream)
{
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: N is negative", fn); return B2K_ERR_INVALID; }
    if (K < 1) { b2k_set_error("%s: K = %d must be at least 1", fn, (int)K); return B2K_ERR_INVALID; }
    if (!(std::isfinite(dt) && dt > 0)) { b2k_set_error("%s: dt = %g must be finite and positive", fn, dt); return B2K_ERR_INVALID; }
    if (!grav) { b2k_set_error("%s: grav is NULL (pass MINUS the robot's gravity, as for accel)", fn); return B2K_ERR_INVALID; }
    if (tau_stride != 0 && tau_stride != (int64_t)K * n) {
        b2k_set_error("%s: tau_stride = %lld must be 0 (one sequence) or K n = %lld (one per trajectory)", fn, (long long)tau_stride,
                      (long long)K * n);
        return B2K_ERR_INVALID;
    }
    if (!A != !B) { b2k_set_error("%s: A and B must both be NULL (states only) or both be given (sensitivities)", fn); return B2K_ERR_INVALID; }
    const int es = dtype == B2K_F64 ? 8 : 4;
    int rc;
    if ((rc = b2k_check_array(fn, "q0", q0, N, es)) || (rc = b2k_check_array(fn, "tau", tau, N, es)) ||
        (rc = b2k_check_array(fn, "q", q, N, es)) || (rc = b2k_check_array(fn, "qd", qd, N, es)))
        return rc;
    if (qd0 && (rc = b2k_check_array(fn, "qd0", qd0, N, es))) return rc;
    const bool sens = A != nullptr;
    if (sens && ((rc = b2k_check_array(fn, "A", A, N, es)) || (rc = b2k_check_array(fn, "B", B, N, es)))) return rc;
    if (N == 0) return B2K_OK;
    const int mode = sens ? B2K_GEN_ACCEL_DERIV : B2K_GEN_ACCEL;
    Program *p = get_program(cache, gen(mode), n, Key(300 + mode, dtype, grav_mask_of(grav), 0));
    if (!p || !p->ok) { b2k_set_error("%s: the rollout kernel could not be built (%s)", fn, p ? p->why.c_str() : "no cache"); return B2K_ERR_INVALID; }
    B2K_ON_DEVICE_OF(q0);
    CUfunction f;
    {
        std::lock_guard<std::mutex> lk(cache->mu);
        if (get_function(p, &f)) { b2k_set_error("%s: %s", fn, p->why.c_str()); return B2K_ERR_CUDA; }
    }
    std::vector<unsigned char> pb = spec_params(p, n, dtype, offset, grav, nullptr);
    // RollP { real h2, h, h6; int K; long long tau_stride; }
    std::vector<unsigned char> rb(3 * es + 4 + 8 + 8, 0);
    const double hv[3] = {dt / 2, dt, dt / 6};
    for (int k = 0; k < 3; k++) {
        if (es == 8) memcpy(&rb[8 * k], &hv[k], 8);
        else { const float v = (float)hv[k]; memcpy(&rb[4 * k], &v, 4); }
    }
    const size_t ko = 3 * es, so = (ko + 4 + 7) & ~(size_t)7;
    memcpy(&rb[ko], &K, 4);
    memcpy(&rb[so], &tau_stride, 8);
    long long nt = N;
    void *args[11] = {pb.data(), rb.data(), (void *)&q0, (void *)&qd0, (void *)&tau, (void *)&q, (void *)&qd, (void *)&A, (void *)&B, (void *)&nt, nullptr};
    const unsigned grid = (unsigned)((N + 63) / 64);
    CUresult cr = driver()->LaunchKernel(f, grid, 1, 1, 64, 1, 1, 0, (CUstream)stream, args, nullptr);
    if (cr != CUDA_SUCCESS) {
        const char *es2 = nullptr;
        driver()->GetErrorString(cr, &es2);
        b2k_set_error("cuLaunchKernel(k_rollout): %s", es2 ? es2 : "?");
        return B2K_ERR_CUDA;
    }
    b2k_count_launch();
    return B2K_OK;
}

extern "C" int b2k_rne_rollout(b2k_rne_t r, int dtype, const void *q0, const void *qd0, int64_t N, int32_t K, double dt,
                               const double *grav, const void *tau, int64_t tau_stride, void *q, void *qd, void *A, void *B, void *stream)
{
    const char *fn = "b2k_rne_rollout";
    if (!r) { b2k_set_error("%s: rne handle is NULL", fn); return B2K_ERR_INVALID; }
    for (int j = 0; j < r->n; j++)
        if ((int)r->L[j][4] != 0) { b2k_set_error("%s: joint %d is prismatic; rollouts serve all-revolute arms", fn, j); return B2K_ERR_INVALID; }
    double offset[B2K_MAX_JOINTS];
    for (int j = 0; j < r->n; j++) offset[j] = r->L[j][5];
    const int gm = grav_mask_of(grav);
    return rollout_run(fn, static_cast<SpecCache *>(r->spec), [r, dtype, gm](int mode) { return dh_gen(r, Key(mode, dtype, gm, 0)); },
                       r->n, offset, dtype, q0, qd0, N, K, dt, grav, tau, tau_stride, q, qd, A, B, stream);
}

extern "C" int b2k_tree_rollout(b2k_tree_t t, int dtype, const void *q0, const void *qd0, int64_t N, int32_t K, double dt,
                                const double *grav, const void *tau, int64_t tau_stride, void *q, void *qd, void *A, void *B, void *stream)
{
    const char *fn = "b2k_tree_rollout";
    if (!t) { b2k_set_error("%s: tree handle is NULL", fn); return B2K_ERR_INVALID; }
    const int gm = grav_mask_of(grav);
    return rollout_run(fn, static_cast<SpecCache *>(t->spec), [t, gm](int mode) { return tree_gen(t, mode, gm); }, t->n, nullptr,
                       dtype, q0, qd0, N, K, dt, grav, tau, tau_stride, q, qd, A, B, stream);
}
