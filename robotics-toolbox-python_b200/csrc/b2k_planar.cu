// b2k_planar.cu -- planar (2-D) forward kinematics and Jacobians of an ETS2 chain: ETS2.eval / fkine / jacob0 /
// jacobe / fkine_jacob0 (reference ET2 and ETS2, src/roboticstoolbox/robot/ET.py and ETS.py, where the walk is a Python
// loop of 3x3 numpy products and jacob0 evaluates a sub-chain FK twice per column).
//
// The chain is the one b2k_chain_create compiles from the ETS2's 3-D embedding (R -> Rz, tx -> tx, ty -> ty, SE2 -> an
// SE3 acting in the xy plane).  The launcher reads it back as a planar table -- per folded constant (cos, sin, x, y),
// per joint axis / flip / jindex -- and rejects a chain that does not stay in the plane before any CUDA call.
//
// One lane per row, a warp per tile of 32 rows (the q tile and the output stages of b2k_fkj.cuh).  The walk keeps the
// pose as (c, s, x, y) in registers: one sincos per revolute joint and a few FMAs per transform, against the 3x3
// rotation products of the 3-D walk.  Per joint it keeps the joint's origin (revolute) or its signed direction of
// travel (prismatic); the columns are formed once the tool is on:
//     R  : sigma (-(y_e - y_j), x_e - x_j, 1)        tx : sigma (cos th_j, sin th_j, 0)      ty : sigma (-sin th_j, cos th_j, 0)
// T (9 reals, row-major 3x3) and J (3n reals, rows vx, vy, w) are staged per warp and leave as the warp's contiguous
// rows.  Every product is written as explicit fma / mul, so each kernel variant rounds the same way and the fused call
// equals the separate ones bit for bit.
#include <math.h>
#include <string.h>

#include "b2k_common.cuh"
#include "b2k_fkj.cuh" // q tile staging (load_q_tile, fkj_qmode, fkj_q_bytes) and the per-warp output stage (TileStage)
#include "b2k_trig.cuh"

template <typename real, int N>
struct PlanarP {
    real C[N + 1][4]; // constant before joint j as (cos, sin, x, y); C[N] is the tail with the tool folded in
    real B[4];        // base, applied to the pose only
    int has_base;
    int axis[N]; // B2K_RZ / B2K_TX / B2K_TY
    int flip[N];
    int jidx[N];
    TrigC<real> trig;
};

template <typename real>
struct Pose2 {
    real c, s, x, y; // [[c, -s, x], [s, c, y], [0, 0, 1]]
};

// P <- P * A, A = (cos, sin, x, y)
template <typename real>
__device__ __forceinline__ void p2_mul_right(Pose2<real> &P, const real *A)
{
    const real x = fma(P.c, A[2], fma(-P.s, A[3], P.x));
    const real y = fma(P.s, A[2], fma(P.c, A[3], P.y));
    const real c = fma(P.c, A[0], -(P.s * A[1]));
    const real s = fma(P.s, A[0], P.c * A[1]);
    P.c = c; P.s = s; P.x = x; P.y = y;
}

// P <- A * P
template <typename real>
__device__ __forceinline__ void p2_mul_left(Pose2<real> &P, const real *A)
{
    const real x = fma(A[0], P.x, fma(-A[1], P.y, A[2]));
    const real y = fma(A[1], P.x, fma(A[0], P.y, A[3]));
    const real c = fma(A[0], P.c, -(A[1] * P.s));
    const real s = fma(A[1], P.c, A[0] * P.s);
    P.c = c; P.s = s; P.x = x; P.y = y;
}

template <typename real, int N, bool WT, bool WJ, int FRAME>
__global__ void __launch_bounds__(B2K_THREADS)
k_planar(const __grid_constant__ PlanarP<real, N> P, const real *__restrict__ q, long long nrows, int ldq, float inv_ldq,
         int qmode, real *__restrict__ Tout, real *__restrict__ Jout, int warp_smem_bytes, int q_bytes)
{
    typedef TileStage<real, 9> TS;
    typedef TileStage<real, 3 * N> JS;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const long long tile = (long long)blockIdx.x * B2K_WARPS_PER_BLOCK + warp;
    const long long row0 = tile << 5;
    if (row0 >= nrows) return;
    const int rows_here = (int)((nrows - row0) < 32 ? (nrows - row0) : 32);
    unsigned char *wbase = smem_raw + (size_t)warp * warp_smem_bytes;
    real *sq = reinterpret_cast<real *>(wbase);
    unsigned char *st_t = wbase + q_bytes;
    unsigned char *st_j = st_t + (WT ? TS::BYTES : 0);
    const int ldqs = qmode ? ldq : (ldq | 1);
    load_q_tile<real>(sq, q + row0 * ldq, rows_here, ldq, inv_ldq, qmode, lane);
    cp_async_wait_all();
    __syncwarp();
    const real *myq = sq + (lane < rows_here ? lane : 0) * ldqs;

    Pose2<real> E = {P.C[0][0], P.C[0][1], P.C[0][2], P.C[0][3]};
    real ka[WJ ? N : 1], kb[WJ ? N : 1]; // per joint: origin (revolute) or signed unit direction of travel (prismatic)
#pragma unroll
    for (int j = 0; j < N; j++) {
        if (j > 0) p2_mul_right(E, P.C[j]);
        const real sg = P.flip[j] ? (real)-1 : (real)1;
        const real eta = sg * myq[P.jidx[j]];
        const int ax = P.axis[j];
        if (ax == B2K_RZ) {
            if (WJ) { ka[j] = E.x; kb[j] = E.y; }
            real sn, cs;
            b2k_sincos(eta, P.trig, &sn, &cs);
            const real c = fma(E.c, cs, -(E.s * sn));
            const real s = fma(E.s, cs, E.c * sn);
            E.c = c; E.s = s;
        } else {
            const real dx = ax == B2K_TX ? E.c : -E.s, dy = ax == B2K_TX ? E.s : E.c;
            if (WJ) { ka[j] = sg * dx; kb[j] = sg * dy; }
            E.x = fma(dx, eta, E.x);
            E.y = fma(dy, eta, E.y);
        }
    }
    p2_mul_right(E, P.C[N]);

    bool async_out = false;
    if (WT) {
        Pose2<real> Tb = E;
        if (P.has_base) p2_mul_left(Tb, P.B);
        const real row[9] = {Tb.c, -Tb.s, Tb.x, Tb.s, Tb.c, Tb.y, (real)0, (real)0, (real)1};
        TS::put_row(st_t, lane, row);
        real *gout = Tout + row0 * 9;
        if (TS::drain_async(st_t, gout, rows_here, lane)) async_out = true;
        else { __syncwarp(); TS::drain(st_t, gout, rows_here, lane); }
    }
    if (WJ) {
        real row[3 * N];
#pragma unroll
        for (int j = 0; j < N; j++) {
            real vx, vy, w;
            if (P.axis[j] == B2K_RZ) {
                const real sg = P.flip[j] ? (real)-1 : (real)1;
                vx = sg * (kb[j] - E.y);
                vy = sg * (E.x - ka[j]);
                w = sg;
            } else {
                vx = ka[j];
                vy = kb[j];
                w = (real)0;
            }
            if (FRAME == 1) { // blkdiag(R^T, 1) of the pose's rotation R
                const real ex = fma(E.c, vx, E.s * vy);
                const real ey = fma(E.c, vy, -(E.s * vx));
                vx = ex; vy = ey;
            }
            row[j] = vx;
            row[N + j] = vy;
            row[2 * N + j] = w;
        }
        JS::put_row(st_j, lane, row);
        real *gout = Jout + row0 * (3 * N);
        if (JS::drain_async(st_j, gout, rows_here, lane)) async_out = true;
        else { __syncwarp(); JS::drain(st_j, gout, rows_here, lane); }
    }
    if (async_out) TS::wait_all(); // the bulk copies read this warp's shared memory: they must finish before the block may retire
}

// ------------------------------------------------------------------ host side
namespace {

// what keeps a 3x4 affine constant from acting in the xy plane as [[c, -s, x], [s, c, y]], or NULL.  The out-of-plane
// entries are tested exactly (the embedding of an SE2 and every product of such embeddings keep them exactly 0 / 1);
// the in-plane block to a few ulp, since the host compiler may fuse the products of a folded constant differently for
// its two off-diagonal entries.
const char *planar_defect(const double *A)
{
    if (A[2] != 0.0 || A[6] != 0.0 || A[8] != 0.0 || A[9] != 0.0 || A[10] != 1.0) return "an out-of-plane rotation";
    if (A[11] != 0.0) return "a non-zero z translation";
    const double tol = 8 * 2.220446049250313e-16 * (fabs(A[0]) + fabs(A[1]) + fabs(A[4]) + fabs(A[5]));
    if (fabs(A[1] + A[4]) > tol || fabs(A[0] - A[5]) > tol) return "an in-plane part that is not a scaled rotation [[c, -s], [s, c]]";
    return nullptr;
}

const char *axis_name(int a)
{
    static const char *names[6] = {"Rx", "Ry", "Rz", "tx", "ty", "tz"};
    return (a >= 0 && a < 6) ? names[a] : "?";
}

// row-major 3x3 SE(2) -> 3x4 SE(3) acting in the xy plane
void embed33(const double *M, double *A)
{
    const double a[12] = {M[0], M[1], 0.0, M[2], M[3], M[4], 0.0, M[5], 0.0, 0.0, 1.0, 0.0};
    memcpy(A, a, sizeof(a));
}

void planar_entry(const double *A, double *out)
{
    out[0] = 0.5 * (A[0] + A[5]);
    out[1] = 0.5 * (A[4] - A[1]);
    out[2] = A[3];
    out[3] = A[7];
}

template <typename real, int N>
void planar_fill(const b2k_chain_s *c, const double *base, const double *tool, PlanarP<real, N> &P)
{
    double e[4], tail[12];
    memcpy(tail, c->A[N], sizeof(tail));
    if (tool) {
        double t[12];
        embed33(tool, t);
        b2k_mul34(c->A[N], t, tail);
    }
    for (int j = 0; j <= N; j++) {
        planar_entry(j == N ? tail : c->A[j], e);
        for (int k = 0; k < 4; k++) P.C[j][k] = (real)e[k];
    }
    P.has_base = 0;
    for (int k = 0; k < 4; k++) P.B[k] = k == 0 ? (real)1 : (real)0;
    if (base) {
        double b[12];
        embed33(base, b);
        planar_entry(b, e);
        for (int k = 0; k < 4; k++) P.B[k] = (real)e[k];
        P.has_base = !(e[0] == 1.0 && e[1] == 0.0 && e[2] == 0.0 && e[3] == 0.0);
    }
    for (int j = 0; j < N; j++) { P.axis[j] = c->axis[j]; P.flip[j] = c->flip[j]; P.jidx[j] = c->jidx[j]; }
    b2k_fill_trig<real>(P.trig);
}

template <typename real, int N>
int planar_launch_n(const b2k_chain_s *c, const double *base, const double *tool, int frame, const real *q, long long nrows,
                    int ldq, real *T, real *J, cudaStream_t st)
{
    PlanarP<real, N> P;
    planar_fill<real, N>(c, base, tool, P);
    const int qb = (int)fkj_q_bytes<real>(ldq);
    const float inv_ldq = 1.0f / (float)ldq;
    const int qmode = fkj_qmode<real>(q, ldq);
    const long long ntiles = (nrows + 31) / 32;
    const long long grid = (ntiles + B2K_WARPS_PER_BLOCK - 1) / B2K_WARPS_PER_BLOCK;
    if (grid > 0x7fffffffLL) { b2k_set_error("b2k_fkine_planar: batch too large for one launch"); return B2K_ERR_INVALID; }
    auto launch = [&](auto kern, bool wt, bool wj) -> int {
        const int wsm = qb + (wt ? TileStage<real, 9>::BYTES : 0) + (wj ? TileStage<real, 3 * N>::BYTES : 0);
        const size_t smem = (size_t)wsm * B2K_WARPS_PER_BLOCK;
        const int per_sm = b2k_blocks_per_sm((const void *)kern, B2K_THREADS, smem);
        if (per_sm < 1) return per_sm < 0 ? per_sm : (b2k_set_error("b2k_fkine_planar: kernel does not fit on an SM (smem %zu B)", smem), B2K_ERR_INVALID);
        kern<<<(unsigned)grid, B2K_THREADS, smem, st>>>(P, q, nrows, ldq, inv_ldq, qmode, T, J, wsm, qb);
        b2k_count_launch();
        B2K_CUDA(cudaGetLastError());
        return B2K_OK;
    };
    if (T && J) return frame ? launch(k_planar<real, N, true, true, 1>, true, true) : launch(k_planar<real, N, true, true, 0>, true, true);
    if (T) return launch(k_planar<real, N, true, false, 0>, true, false);
    return frame ? launch(k_planar<real, N, false, true, 1>, false, true) : launch(k_planar<real, N, false, true, 0>, false, true);
}

// B2K_OK when the chain (and the base / tool, row-major 3x3, either may be NULL) is planar; otherwise an error naming the
// first transform, in chain order, that leaves the plane.  Host only.
int planar_check(const char *fn, const b2k_chain_s *c, const double *base, const double *tool)
{
    const double *M[2] = {base, tool};
    const char *names[2] = {"base", "tool"};
    for (int k = 0; k < 2; k++) {
        if (!M[k]) continue;
        if (M[k][6] != 0.0 || M[k][7] != 0.0 || M[k][8] != 1.0) {
            b2k_set_error("%s: %s is not an SE(2) matrix (bottom row must be 0 0 1)", fn, names[k]);
            return B2K_ERR_INVALID;
        }
        double A[12];
        embed33(M[k], A);
        if (const char *d = planar_defect(A)) { b2k_set_error("%s: %s has %s", fn, names[k], d); return B2K_ERR_INVALID; }
    }
    for (int j = 0; j <= c->n; j++) {
        if (const char *d = planar_defect(c->A[j])) {
            if (j < c->n) b2k_set_error("%s: the chain is not planar: the constant before joint %d has %s", fn, j, d);
            else b2k_set_error("%s: the chain is not planar: the constant after the last joint has %s", fn, d);
            return B2K_ERR_INVALID;
        }
        if (j < c->n && c->axis[j] != B2K_RZ && c->axis[j] != B2K_TX && c->axis[j] != B2K_TY) {
            b2k_set_error("%s: the chain is not planar: joint %d is %s (planar joints are Rz, tx and ty)", fn, j, axis_name(c->axis[j]));
            return B2K_ERR_INVALID;
        }
    }
    return B2K_OK;
}

} // namespace

extern "C" int b2k_fkine_planar(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *base,
                                const double *tool, int frame, void *T, void *J, void *stream)
{
    const char *fn = "b2k_fkine_planar";
    int rc = b2k_check_chain(fn, c, dtype, q, N, ldq);
    if (rc) return rc;
    if (frame != 0 && frame != 1) { b2k_set_error("%s: frame must be 0 (jacob0) or 1 (jacobe), got %d", fn, frame); return B2K_ERR_INVALID; }
    if (!T && !J) { b2k_set_error("%s: T and J are both NULL; nothing to compute", fn); return B2K_ERR_INVALID; }
    if ((rc = planar_check(fn, c, base, tool))) return rc;
    // T and J leave through per-warp stages of 9- and 3n-element rows (TileStage in b2k_fkj.cuh)
    const int es = dtype == B2K_F64 ? 8 : 4;
    if ((T && (rc = b2k_check_array(fn, "T", T, N, b2k_stage_unit(9 * es)))) ||
        (J && (rc = b2k_check_array(fn, "J", J, N, b2k_stage_unit(3 * c->n * es)))))
        return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(q);
    cudaStream_t st = (cudaStream_t)stream;
    return b2k_for_joints(c->n, [&](auto n) {
        return dtype == B2K_F64 ? planar_launch_n<double, n.value>(c, base, tool, frame, (const double *)q, N, (int)ldq,
                                                                   (double *)T, (double *)J, st)
                                : planar_launch_n<float, n.value>(c, base, tool, frame, (const float *)q, N, (int)ldq,
                                                                  (float *)T, (float *)J, st);
    });
}
