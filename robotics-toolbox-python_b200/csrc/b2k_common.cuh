// b2k_common.cuh -- shared types between the host-side chain compiler and the sm_90a kernels.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/b2kin.h"

#define B2K_WARPS_PER_BLOCK 4
#define B2K_THREADS (32 * B2K_WARPS_PER_BLOCK)

// Structure classes of a folded SE(3) constant A = [Ra | ta] (exact 0/1 pattern tests on the
// host, so the specialised device paths are bit-identical to the general product).
enum : int {
    AK_IDENT = 0, // Ra = I
    AK_RX = 1,    // Ra = [[1,0,0],[0,a,b],[0,c,d]]
    AK_RY = 2,    // Ra = [[a,0,b],[0,1,0],[c,0,d]]
    AK_RZ = 3,    // Ra = [[a,b,0],[c,d,0],[0,0,1]]
    AK_GEN = 4,   // anything else
    AK_ROTMASK = 7,
    AK_TX = 8, // ta.x != 0
    AK_TY = 16,
    AK_TZ = 32
};

// Constants of the in-house sincos (b2k_trig.cuh).  They live in the kernel-parameter constant
// bank so every polynomial coefficient is an immediate c[0x0][..] operand of an FMA; literal
// doubles would each cost two MOV-immediate instructions on the uniform datapath.
template <typename real>
struct TrigC {
    real two_over_pi, magic, pio2_hi, pio2_mid, pio2_lo, fast_limit;
    real s[6]; // sin(r) = r + r^3 (s0 + z s1 + ... ), z = r^2
    real c[6]; // cos(r) = 1 - z/2 + z^2 (c0 + z c1 + ...)
};

template <typename real>
inline void b2k_fill_trig(TrigC<real> &t);
template <>
inline void b2k_fill_trig<double>(TrigC<double> &t)
{
    t.two_over_pi = 0.6366197723675814;
    t.magic = 6755399441055744.0; // 1.5 * 2^52: adds k = rint(x 2/pi) into the low mantissa bits
    t.pio2_hi = 1.5707963267948966;
    t.pio2_mid = 6.123233995736766e-17;
    t.pio2_lo = -1.4973849048591698e-33;
    t.fast_limit = 105615.0; // same validity bound CUDA's own three-FMA reduction uses
    const double s[6] = {-1.66666666666666324348e-01, 8.33333333332248946124e-03, -1.98412698298579493134e-04,
                         2.75573137070700676789e-06, -2.50507602534068634195e-08, 1.58969099521155010221e-10};
    const double c[6] = {4.16666666666666019037e-02, -1.38888888888741095749e-03, 2.48015872894767294178e-05,
                         -2.75573143513906633035e-07, 2.08757232129817482790e-09, -1.13596475577881948265e-11};
    for (int i = 0; i < 6; i++) { t.s[i] = s[i]; t.c[i] = c[i]; }
}
template <>
inline void b2k_fill_trig<float>(TrigC<float> &t)
{
    t.two_over_pi = 0.6366197723675814f;
    t.magic = 12582912.0f; // 1.5 * 2^23
    t.pio2_hi = 1.5707963705062866f;
    t.pio2_mid = -4.371138828673793e-08f;
    t.pio2_lo = -1.7151245100058819e-15f;
    t.fast_limit = 105615.0f;
    const float s[6] = {-1.6666654611e-1f, 8.3321608736e-3f, -1.9515295891e-4f, 0.f, 0.f, 0.f};
    const float c[6] = {4.166664568298827e-2f, -1.388731625493765e-3f, 2.443315711809948e-5f, 0.f, 0.f, 0.f};
    for (int i = 0; i < 6; i++) { t.s[i] = s[i]; t.c[i] = c[i]; }
}

// Device-side chain: n steps of (constant A_j, joint j) followed by a tail constant A_n.
// Passed BY VALUE as a __grid_constant__ kernel parameter so every entry is a constant-bank
// operand (no loads in the unrolled chain walk).
template <typename real, int N>
struct ChainP {
    real A[N + 1][12]; // row-major 3x4: r00 r01 r02 tx | r10 r11 r12 ty | r20 r21 r22 tz
    real B[12];        // base, applied to the pose only (reference RobotKinematics.py:94 vs :158)
    int akind[N + 1];
    int axis[N];  // B2K_RX..B2K_TZ
    int flip[N];  // 0 / 1
    int jidx[N];  // column of q
    int has_base; // 0: B is identity
    int all_rz;   // every joint is an unflipped Rz
    TrigC<real> trig;
};

// Host-side compiled chain (fp64 master copy); see b2k_chain.cu.
struct b2k_chain_s {
    int n, m, q_width;
    double A[B2K_MAX_JOINTS + 1][12];
    int axis[B2K_MAX_JOINTS];
    int flip[B2K_MAX_JOINTS];
    int jidx[B2K_MAX_JOINTS];
    double qlim_l[B2K_MAX_JOINTS];
    double qlim_h[B2K_MAX_JOINTS];
    int all_rz;
    int dh_like;      // all_rz and every inter-joint constant A_1..A_{n-1} has the Rx form (or is a pure translation)
    int dense_jindex; // jidx[j] == j for all j
    int distinct_jindex; // no two joints read the same column of q
};

// One call of b2k_ik_lm, b2k_ikine_null or b2k_ikine_qp as the host passes it to the launchers (b2k_ik.cuh), after
// ik_dispatch (b2k_api.cu) has validated it.  Tep .. residual are device arrays of N rows; we and gains.pi are host.
struct IkArgs {
    const void *Tep, *q0;
    void *q_out;
    int *success, *iterations, *searches;
    void *residual;
    long long N;
    int ilimit, slimit;
    double tol;
    int reject_jl;
    const double *we;
    double lambda;
    int method;
    unsigned long long seed;
    int semantics, rng_per_row;
    // the gains and band of the null-space terms (kq, km, ps, pi) and of the QP step (all six); pi holds n values
    struct {
        double kj, ks, kq, km, ps;
        const double *pi;
    } gains;
};

// what an fkj call (b2k_fkj.cuh) writes: the pose T, the Jacobian in the start frame, or in the end-effector frame
enum { FKJ_T = 1, FKJ_J0 = 2, FKJ_JE = 4 };

// the unit a per-warp output stage of rows of `row_bytes` is copied in (TileStage<real, n>::UB in b2k_fkj.cuh): 16 bytes
// when a row is a whole number of 16-byte units, else 8, else 4.  An output array must be aligned to it.
constexpr int b2k_stage_unit(int row_bytes) { return row_bytes % 16 == 0 ? 16 : (row_bytes % 8 == 0 ? 8 : 4); }

struct b2k_rne_s {
    int n, mdh;
    double L[B2K_MAX_JOINTS][24];
    void *spec; // cache of run-time compiled, robot-specialised kernels (b2k_rne_spec.cu)
};

// Operations on an rne handle.  B2K_GEN_RNE..B2K_GEN_RNE_WRENCH are served by the robot-specialised kernels
// (b2k_rne_gen.cpp, b2k_rne_spec.cu) on the full 32-row tiles and by the generic ones (b2k_rne.cuh) on the rest; the
// derivatives of DH arms only by the generic ones, those of trees by the generated kernels.  RNE..ACCEL, RNE_DERIV and
// ACCEL_DERIV are also the public B2K_DYN_* codes of the tree entry points.  The regressors are one operation per robot
// kind: RNE_REGRESSOR (DH arms, 14 parameters per link, generic kernel only) is no tree operation, and TREE_REGRESSOR
// (B2K_DYN_REGRESSOR: trees, 10 parameters per joint group, generated kernel only) is no DH operation; each robot kind's
// entry points reject the other's code.
enum { B2K_GEN_RNE = 0, B2K_GEN_INERTIA = 1, B2K_GEN_GRAVLOAD = 2, B2K_GEN_ITORQUE = 3, B2K_GEN_CORIOLIS = 4, B2K_GEN_ACCEL = 5,
       B2K_GEN_RNE_WRENCH = 6, B2K_GEN_RNE_DERIV = 7, B2K_GEN_ACCEL_DERIV = 8, B2K_GEN_RNE_REGRESSOR = 9,
       B2K_GEN_TREE_REGRESSOR = 10, B2K_GEN_NOPS = 11 };
static_assert(B2K_GEN_RNE == B2K_DYN_RNE && B2K_GEN_INERTIA == B2K_DYN_INERTIA && B2K_GEN_GRAVLOAD == B2K_DYN_GRAVLOAD &&
                  B2K_GEN_ITORQUE == B2K_DYN_ITORQUE && B2K_GEN_CORIOLIS == B2K_DYN_CORIOLIS && B2K_GEN_ACCEL == B2K_DYN_ACCEL &&
                  B2K_GEN_RNE_DERIV == B2K_DYN_RNE_DERIV && B2K_GEN_ACCEL_DERIV == B2K_DYN_ACCEL_DERIV &&
                  B2K_GEN_TREE_REGRESSOR == B2K_DYN_REGRESSOR,
              "B2K_DYN_* (b2kin.h) are the B2K_GEN_* codes of the tree operations");

// What an operation reads and writes.  Every input is an (N, n) array; every output has rows of n or n * n reals, except
// the base wrench, the (N, 6) second output of B2K_GEN_RNE_WRENCH, and the regressors, (N, n, k n) with k parameters per
// link (14 DH, 10 tree).
struct b2k_rne_op_s {
    int nin, nout;          // input / output arrays
    bool square;            // output rows of n * n reals
    bool wrench;            // the second output is the base wrench
    bool grav, fext;        // reads the gravity vector / the tip wrench
    const char *in[3], *out[3]; // argument names, as the error messages print them
    int regressor = 0;          // a regressor: parameters per link, output rows of n * regressor * n reals
    constexpr int out_row(int o, int n) const { return regressor ? regressor * n * n : (wrench && o == 1 ? 6 : (square ? n * n : n)); }
};
inline constexpr b2k_rne_op_s B2K_RNE_OPS[B2K_GEN_NOPS] = {
    {3, 1, false, false, true, true, {"q", "qd", "qdd"}, {"tau"}},                                     // RNE
    {1, 1, true, false, false, false, {"q"}, {"output"}},                                             // INERTIA
    {1, 1, false, false, true, false, {"q"}, {"output"}},                                             // GRAVLOAD
    {2, 1, false, false, false, false, {"q", "second input"}, {"output"}},                            // ITORQUE
    {2, 1, true, false, false, false, {"q", "second input"}, {"output"}},                             // CORIOLIS
    {3, 1, false, false, true, false, {"q", "second input", "third input"}, {"output"}},              // ACCEL
    {3, 2, false, true, true, true, {"q", "qd", "qdd"}, {"tau", "wbase"}},                            // RNE_WRENCH
    {3, 2, true, false, true, true, {"q", "qd", "qdd"}, {"dtau_dq", "dtau_dqd"}},                     // RNE_DERIV
    {3, 3, true, false, true, false, {"q", "qd", "torque"}, {"dqdd_dq", "dqdd_dqd", "dqdd_dtau"}},    // ACCEL_DERIV
    {3, 1, false, false, true, false, {"q", "qd", "qdd"}, {"Y"}, 14},                                 // RNE_REGRESSOR
    {3, 1, false, false, true, false, {"q", "qd", "qdd"}, {"Y"}, 10},                                 // TREE_REGRESSOR
};

// The arrays of one launch of an operation, device pointers: unused entries are NULL
struct b2k_rne_args {
    const void *in[3];
    void *out[3];
    long long nrows;
    const double *grav, *fext;
};

void b2k_rne_spec_attach(b2k_rne_s *r);
void b2k_rne_spec_detach(b2k_rne_s *r);
// mode = B2K_GEN_RNE..B2K_GEN_RNE_WRENCH; returns the rows served by the specialised kernel (a multiple of 32, possibly 0)
// or a negative b2k_status.  out2: the base wrench (nrows, 6) of B2K_GEN_RNE_WRENCH, NULL for every other mode.
long long b2k_rne_spec_launch(const b2k_rne_s *r, int mode, int dtype, const void *in0, const void *in1, const void *in2,
                              long long nrows, const double *grav, const double *fext, void *out, void *out2, cudaStream_t st);
// Y (a.out[0]) of a tree's regressor over a.nrows rows of a.in = q, qd, qdd (b2k_rne_spec.cu): the chunks of
// b2k_tree_regressor_gram, whose arguments are already checked
int b2k_tree_regressor_rows(b2k_tree_t t, int dtype, const b2k_rne_args &a, cudaStream_t st);

// ---- error plumbing and argument checks (b2k_api.cu)
void b2k_set_error(const char *fmt, ...);
// The arguments every entry point that walks a chain shares, in this order: handle, dtype, joint count, N >= 0, q not
// NULL when N > 0, q row width ldq in [q_width, B2K_MAX_QWIDTH], and, when q_on_device, q aligned to its element size
// (a kernel reads it element-wise at worst; the host pointers of the *_host front ends only go through cudaMemcpy).
int b2k_check_chain(const char *fn, const b2k_chain_s *c, int dtype, const void *q, int64_t N, int64_t ldq,
                    bool q_on_device = true);
// an array of N rows: not NULL when N > 0, and aligned to `align` bytes (1: any address)
int b2k_check_array(const char *fn, const char *name, const void *p, int64_t N, unsigned align);
// a host 4x4 row-major matrix, NULL or with the bottom row 0 0 0 1; index >= 0 is printed after the name
int b2k_check_affine(const char *fn, const char *name, const double *M, int index = -1);
int b2k_cuda_fail(cudaError_t e, const char *what);
void b2k_count_launch(int n = 1);
int b2k_num_sms(int *device_out = nullptr);
// resident blocks per SM for (kernel, threads, dynamic smem), cached; also raises the kernel's
// dynamic shared-memory limit.  <0 on CUDA error.
int b2k_blocks_per_sm(const void *func, int threads, size_t smem);
// once per device: keep freed stream-ordered allocations cached in the default memory pool
void b2k_keep_mempool();

// Calls go(std::integral_constant<int, N>()) for the joint count n = N in 1..10: the kernels are unrolled per N.
template <typename F>
int b2k_for_joints(int n, F &&go)
{
    static_assert(B2K_MAX_JOINTS == 10, "one case per joint count");
    switch (n) {
    case 1: return go(std::integral_constant<int, 1>());
    case 2: return go(std::integral_constant<int, 2>());
    case 3: return go(std::integral_constant<int, 3>());
    case 4: return go(std::integral_constant<int, 4>());
    case 5: return go(std::integral_constant<int, 5>());
    case 6: return go(std::integral_constant<int, 6>());
    case 7: return go(std::integral_constant<int, 7>());
    case 8: return go(std::integral_constant<int, 8>());
    case 9: return go(std::integral_constant<int, 9>());
    case 10: return go(std::integral_constant<int, 10>());
    }
    b2k_set_error("unsupported joint count %d", n);
    return B2K_ERR_INVALID;
}

#define B2K_CUDA(call)                                   \
    do {                                                 \
        cudaError_t _e = (call);                         \
        if (_e != cudaSuccess) return b2k_cuda_fail(_e, #call); \
    } while (0)

// Every device-pointer entry point runs on the device that owns its first array argument: a caller
// whose current device is cuda:0 may hand in buffers (and a stream) of cuda:1.  The guard looks the
// pointer up (cudaPointerGetAttributes), switches the calling thread to that device for the duration
// of the call and restores the previous one on every exit path.
struct DeviceGuard {
    int prev = -1;
    bool switched = false;
    int rc = B2K_OK;
    explicit DeviceGuard(const void *devptr) { rc = enter_ptr(devptr); }
    DeviceGuard(int device, bool) { rc = enter(device); }
    ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
    DeviceGuard(const DeviceGuard &) = delete;
    DeviceGuard &operator=(const DeviceGuard &) = delete;
    inline int enter(int device)
    {
        cudaError_t e = cudaGetDevice(&prev);
        if (e != cudaSuccess) return b2k_cuda_fail(e, "cudaGetDevice");
        if (device == prev) return B2K_OK;
        e = cudaSetDevice(device);
        if (e != cudaSuccess) return b2k_cuda_fail(e, "cudaSetDevice");
        switched = true;
        return B2K_OK;
    }
    inline int enter_ptr(const void *p)
    {
        if (!p) return B2K_OK;
        cudaPointerAttributes a;
        cudaError_t e = cudaPointerGetAttributes(&a, p);
        if (e != cudaSuccess) { cudaGetLastError(); return b2k_cuda_fail(e, "cudaPointerGetAttributes"); }
        if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) return enter(a.device);
        if (a.type == cudaMemoryTypeUnregistered) {
            b2k_set_error("array argument %p is not a CUDA device pointer (host arrays go through the *_host entry points)", p);
            return B2K_ERR_INVALID;
        }
        return B2K_OK; // pinned host memory is device-accessible from the current device
    }
};
#define B2K_ON_DEVICE_OF(ptr)  \
    DeviceGuard _guard(ptr);   \
    if (_guard.rc) return _guard.rc

// ---- small host helpers shared by launchers
void b2k_mat_to34(const double *T16, double *A12);          // row-major 4x4 -> 3x4
void b2k_mul34(const double *A, const double *B, double *C); // C = A*B on 3x4 affine
int b2k_classify34(const double *A);
void b2k_ident34(double *A);

template <typename real, int N>
void b2k_fill_chain(const b2k_chain_s *c, const double *base, const double *tool, bool base_into_chain,
                    ChainP<real, N> &P)
{
    double A0[12], An[12], tmp[12];
    for (int j = 0; j <= N; j++)
        for (int k = 0; k < 12; k++) P.A[j][k] = (real)c->A[j][k];
    for (int k = 0; k < 12; k++) { A0[k] = c->A[0][k]; An[k] = c->A[N][k]; }
    double B[12];
    b2k_ident34(B);
    P.has_base = 0;
    if (base) {
        b2k_mat_to34(base, tmp);
        if (base_into_chain) { // pose-only kernels: fold base into the first constant
            b2k_mul34(tmp, A0, B);
            for (int k = 0; k < 12; k++) A0[k] = B[k];
            b2k_ident34(B);
        } else {
            for (int k = 0; k < 12; k++) B[k] = tmp[k];
            P.has_base = (b2k_classify34(B) != AK_IDENT);
        }
    }
    if (tool) {
        b2k_mat_to34(tool, tmp);
        double t2[12];
        if (N == 0) {
            b2k_mul34(A0, tmp, t2);
            for (int k = 0; k < 12; k++) A0[k] = t2[k];
        } else {
            b2k_mul34(An, tmp, t2);
            for (int k = 0; k < 12; k++) An[k] = t2[k];
        }
    }
    for (int k = 0; k < 12; k++) { P.A[0][k] = (real)A0[k]; P.A[N][k] = (real)(N == 0 ? A0[k] : An[k]); P.B[k] = (real)B[k]; }
    for (int j = 0; j <= N; j++) {
        double Aj[12];
        for (int k = 0; k < 12; k++) Aj[k] = (j == 0) ? A0[k] : (j == N ? An[k] : c->A[j][k]);
        P.akind[j] = b2k_classify34(Aj);
    }
    for (int j = 0; j < N; j++) { P.axis[j] = c->axis[j]; P.flip[j] = c->flip[j]; P.jidx[j] = c->jidx[j]; }
    P.all_rz = c->all_rz;
    b2k_fill_trig<real>(P.trig);
}

#ifdef __CUDACC__
// The three used rows of a row-major 4x4 pose (12 reals) as 16-byte vector loads / the whole pose as 16-byte vector
// stores; the caller has checked that the array is 16-byte aligned (any torch allocation is).
template <typename real> __device__ __forceinline__ void load12(const real *p, real *o);
template <> __device__ __forceinline__ void load12<double>(const double *p, double *o)
{
    const double2 *v = reinterpret_cast<const double2 *>(p);
#pragma unroll
    for (int k = 0; k < 6; k++) { const double2 x = __ldg(v + k); o[2 * k] = x.x; o[2 * k + 1] = x.y; }
}
template <> __device__ __forceinline__ void load12<float>(const float *p, float *o)
{
    const float4 *v = reinterpret_cast<const float4 *>(p);
#pragma unroll
    for (int k = 0; k < 3; k++) { const float4 x = __ldg(v + k); o[4 * k] = x.x; o[4 * k + 1] = x.y; o[4 * k + 2] = x.z; o[4 * k + 3] = x.w; }
}

template <typename real> __device__ __forceinline__ void store16(real *p, const real *v);
template <> __device__ __forceinline__ void store16<double>(double *p, const double *v)
{
    double2 *o = reinterpret_cast<double2 *>(p);
#pragma unroll
    for (int k = 0; k < 8; k++) o[k] = make_double2(v[2 * k], v[2 * k + 1]);
}
template <> __device__ __forceinline__ void store16<float>(float *p, const float *v)
{
    float4 *o = reinterpret_cast<float4 *>(p);
#pragma unroll
    for (int k = 0; k < 4; k++) o[k] = make_float4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
}
// element index of an (N, n) array -> (row, axis).  n is a run-time value: the 64-bit division the plain expression
// compiles to is a ~100-instruction software routine per element (it, not the 168 B / row of stores, bounded k_jtraj and
// k_mtraj); arrays below 2^32 elements take the 32-bit division.
__device__ __forceinline__ void split_elem(long long e, int n, long long total, long long &row, int &j)
{
    if (total <= 0xffffffffLL) {
        const unsigned r = (unsigned)e / (unsigned)n;
        row = r;
        j = (int)((unsigned)e - r * (unsigned)n);
    } else {
        row = e / n;
        j = (int)(e - row * n);
    }
}

template <typename real> __device__ __forceinline__ real r_atan2(real y, real x);
template <> __device__ __forceinline__ double r_atan2<double>(double y, double x) { return atan2(y, x); }
template <> __device__ __forceinline__ float r_atan2<float>(float y, float x) { return atan2f(y, x); }
template <typename real> __device__ __forceinline__ real r_eps() { return sizeof(real) == 8 ? (real)2.220446049250313e-16 : (real)1.1920929e-07f; }

// spatialmath's tr2eul: R = Rz(phi) Ry(theta) Rz(psi) -> (phi, theta, psi), theta >= 0; FLIP takes the other solution
// (phi + pi, theta < 0).  With |R02| and |R12| below 10 eps phi is 0.  Used by jacob0_analytical("eul") and ikine_a.
// SinCos, when given, is a stateless functor SinCos()(x, s, c) that forms sin and cos of phi (a caller whose angles are
// small can avoid libm's Payne-Hanek branch); by default libm's sin and cos.
template <typename real, bool FLIP = false, typename SinCos = void>
__device__ __forceinline__ void rot_to_eul(const real R[3][3], real g[3])
{
    real sp = 0, cp = 1;
    if (fabs(R[0][2]) < 10 * r_eps<real>() && fabs(R[1][2]) < 10 * r_eps<real>()) g[0] = 0;
    else {
        g[0] = FLIP ? r_atan2<real>(-R[1][2], -R[0][2]) : r_atan2<real>(R[1][2], R[0][2]);
        if constexpr (std::is_void<SinCos>::value) { sp = sin(g[0]); cp = cos(g[0]); }
        else SinCos()(g[0], sp, cp);
    }
    g[1] = r_atan2<real>(cp * R[0][2] + sp * R[1][2], R[2][2]);
    g[2] = r_atan2<real>(-sp * R[0][0] + cp * R[1][0], -sp * R[0][1] + cp * R[1][1]);
}
#endif // __CUDACC__
