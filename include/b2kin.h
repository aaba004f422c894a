/*
 * b2kin.h -- C ABI of libb2kin.so: batched serial-chain kinematics / dynamics on H100 (sm_90a).
 *
 * This is the drop-in boundary for the reference's native fast path
 * (petercorke/robotics-toolbox-python, src/roboticstoolbox/core/).  Each entry point names
 * the reference interface it replaces (file:line relative to the reference repo).  The
 * reference boundary is two CPython extension modules taking PyObject tuples and PyCapsule
 * handles (fknm.cpp:23-93, frne.c:42-62); this one is plain C: POD arguments, opaque handles,
 * no Python.h, no torch types.  INTEGRATION.md shows the ctypes binding a reference maintainer
 * would add.
 *
 * Conventions
 *   - every batched array is a DEVICE pointer, contiguous, row-major:
 *       q (N, ldq)   T (N,4,4)   J (N,6,n)   tau (N,n)   Tep (N,4,4)
 *     i.e. the values of numpy.asarray(reference_result) for row i of the batch
 *     (reference batch FK layout: fknm.cpp:1005,1048-1051; single-q results are F-ordered
 *     there, fknm.cpp:993,813 -- same values, different strides).
 *   - small per-call constants (base, tool, gravity, fext, mask) are HOST pointers, fp64,
 *     4x4 matrices row-major; NULL means "not given" exactly like None in the reference.
 *   - dtype selects the arithmetic type of the device arrays: B2K_F32 or B2K_F64.
 *   - stream is a cudaStream_t passed as void* (NULL = legacy default stream).  All compute
 *     entry points are asynchronous on that stream.
 *   - every function returns 0 on success, a negative b2k_status otherwise; the message for
 *     the calling thread is available from b2k_last_error().
 *   - handles are immutable after creation: safe to use from many host threads / streams
 *     (the reference's frne capsule is mutated per call, frne.c:142-153,193-207).
 */
#ifndef B2KIN_H
#define B2KIN_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2K_VERSION 100 /* 0.1.0 */

#define B2K_F32 0
#define B2K_F64 1

/* largest number of joints a chain / DH robot may have (kernels are unrolled per n) */
#define B2K_MAX_JOINTS 10
/* largest q row width (max jindex + 1); reference: q may be wider than n, methods.cpp:338 */
#define B2K_MAX_QWIDTH 16

/* elementary-transform axis codes, as reference ET.py:244-266 */
#define B2K_RX 0
#define B2K_RY 1
#define B2K_RZ 2
#define B2K_TX 3
#define B2K_TY 4
#define B2K_TZ 5

/* LM damping rule, reference ik.cpp:157-209 / IK.py:997-1005 */
#define B2K_LM_CHAN 0     /* Wn = lambda * E * I   */
#define B2K_LM_WAMPLER 1  /* Wn = lambda * I       */
#define B2K_LM_SUGIHARA 2 /* Wn = (E + lambda) * I */
/* the other two solvers of the fknm module ride the same loop and entry point (method argument of b2k_ik_lm) */
#define B2K_IK_NR 3 /* Newton-Raphson, dq = pinv_d(J) e, lambda = pinv_damping: fknm.IK_NR_c, ik.cpp:121-155 */
#define B2K_IK_GN 4 /* Gauss-Newton, min-norm solution of (J^T We J) dq = J^T We e: fknm.IK_GN_c, ik.cpp:79-119 */

/* which of the reference's two LM loops to reproduce */
#define B2K_IK_SEM_CPP 0    /* fknm.IK_LM_c -> _IK_loop, ik.cpp:19-75 (ETS.ik_LM)       */
#define B2K_IK_SEM_PYTHON 1 /* IKSolver._solve + IK_LM.step, IK.py:297-367,994-1017 (ETS.ikine_LM) */

typedef enum {
    B2K_OK = 0,
    B2K_ERR_INVALID = -1, /* bad argument (shape, dtype, NULL, n too large, ...) */
    B2K_ERR_CUDA = -2,    /* a CUDA runtime call failed; message carries cudaGetErrorString */
    B2K_ERR_ALLOC = -3
} b2k_status;

typedef struct b2k_chain_s *b2k_chain_t; /* replaces the "ETS" PyCapsule, structs.h:25-56 */
typedef struct b2k_rne_s *b2k_rne_t;     /* replaces the "Robot" PyCapsule, frne.h            */
typedef struct b2k_tree_s *b2k_tree_t;   /* a rigid-body tree as Robot.rne walks it, Robot.py:1704-1903 */

const char *b2k_last_error(void);
int b2k_version(void);

/* ---------------------------------------------------------------- chain description
 * Replaces fknm.ET_init + fknm.ETS_init (fknm.cpp:1182-1239, 1066-1114; Python side
 * ET.py:100-125, ETS.py:62-69).  m elementary transforms, in chain order:
 *   isjoint[i]  1 = variable joint, 0 = constant
 *   axis[i]     B2K_RX..B2K_TZ (joints only)
 *   flip[i]     1 = joint moves in the opposite direction (eta = -q)
 *   jindex[i]   column of q this joint reads (joints only)
 *   T[i*16..]   constant 4x4, row-major (constants only; ignored for joints)
 *   qlim[i*2..] joint limits low/high (joints only; the caller applies the reference defaults
 *               [-pi,pi] / [0,1], ET.py:109-115)
 * All constants are copied (the reference keeps a borrowed pointer, fknm.cpp:1207).
 * Runs of constants are folded into one SE(3) constant per joint on the host -- the
 * reference's own ETS.compile() rule, ETS.py:857-906.
 */
int b2k_chain_create(int m, const int32_t *isjoint, const int32_t *axis, const int32_t *flip,
                     const int32_t *jindex, const double *T, const double *qlim,
                     b2k_chain_t *out);
int b2k_chain_destroy(b2k_chain_t chain);
/* n = joints, m = elementary transforms, q_width = max jindex + 1 */
int b2k_chain_info(b2k_chain_t chain, int *n, int *m, int *q_width);

/* ---------------------------------------------------------------- entry points that walk a chain
 * b2k_fkine, b2k_fkine_frames, b2k_jacob0, b2k_jacobe, b2k_fkine_jacob0, b2k_fkine_jacobe, b2k_fkine_planar,
 * b2k_gravjac, b2k_pay, b2k_paycap and the host front ends b2k_fkine_host and b2k_fkine_jacob0_host take a chain handle
 * and q (N, ldq), q_width <= ldq <= B2K_MAX_QWIDTH.  Every argument is checked before any CUDA call, in this order: the
 * chain handle, dtype, N >= 0, q, ldq; then the entry point's own scalars and host tables; then its device arrays in
 * argument order.  A device array may be NULL only when N = 0 (T or J of b2k_fkine_planar: when not wanted), and must
 * be aligned as follows (NULL counts as aligned):
 *   q                                  its element size
 *   T of the fkj calls, out of frames  32 bytes
 *   J of the fkj calls                 the piece a row of 6n elements is copied in: 16 bytes when the row is a
 *                                      multiple of 16 bytes, else 8 when a multiple of 8, else 4 (fp64: 16; fp32:
 *                                      16 for even n, else 8)
 *   T, J of b2k_fkine_planar           the same rule on rows of 9 and 3n elements
 *   static-force arrays                their element size (joint: 4 bytes)
 * The host front ends take host arrays and need no alignment.  N = 0 returns B2K_OK without touching a device. */

/* ---------------------------------------------------------------- forward kinematics
 * Replaces fknm.ETS_fkine (fknm.cpp:923-1064 -> _ETS_fkine methods.cpp:318-352):
 *   T[i] = base * prod_k ET_k(q[i, jindex_k]) * tool
 * ldq = row stride of q in elements (>= q_width).
 */
int b2k_fkine(b2k_chain_t chain, int dtype, const void *q, int64_t N, int64_t ldq,
              const double *base, const double *tool, void *T, void *stream);

/* The poses of several frames along one chain from a single walk: the device side of fkine_all (reference
 * Robot.fkine_all, Robot.py:638-700, and DHRobot.fkine_all, DHRobot.py:1018-1064: Python loops over the links).
 * Frame k is  base * A_0 J_0(q) ... J_after[k](q) * tails[k]  -- the pose right after joint after[k] (0-based position
 * of the joint along the chain) times a constant 4x4 (row-major, host) -- or, for after[k] = -1, the constant tails[k]
 * itself (the base frame, links that depend on no joint; the caller multiplies the base in).  after[] ascending.
 * out is (N, nslots, 4, 4) row-major; frame k goes to slot[k] of every row; slots not named are left
 * untouched (a branched robot takes one call per branch into the same array).  The chain's tool constant and the
 * transforms behind its last joint do not enter. */
int b2k_fkine_frames(b2k_chain_t chain, int dtype, const void *q, int64_t N, int64_t ldq, const double *base,
                     int nframes, const int32_t *after, const int32_t *slot, const double *tails, void *out,
                     int64_t nslots, void *stream);

/* Replaces fknm.ETS_jacob0 (fknm.cpp:785-850 -> _ETS_jacob0 methods.cpp:112-216), batched:
 * J[i] = geometric Jacobian in the chain's start frame, (6,n) row-major per row; no base
 * (reference RobotKinematics.py:158), tool included. */
int b2k_jacob0(b2k_chain_t chain, int dtype, const void *q, int64_t N, int64_t ldq,
               const double *tool, void *J, void *stream);

/* Replaces fknm.ETS_jacobe (fknm.cpp:852-921 -> _ETS_jacobe methods.cpp:219-316), batched:
 * Jacobian in the end-effector frame. */
int b2k_jacobe(b2k_chain_t chain, int dtype, const void *q, int64_t N, int64_t ldq,
               const double *tool, void *J, void *stream);

/* Fused pose + base-frame Jacobian in one pass over q (the BASELINE headline op):
 * T as b2k_fkine (base and tool applied), J as b2k_jacob0 (tool applied, no base). */
int b2k_fkine_jacob0(b2k_chain_t chain, int dtype, const void *q, int64_t N, int64_t ldq,
                     const double *base, const double *tool, void *T, void *J, void *stream);

/* Fused pose + end-effector-frame Jacobian. */
int b2k_fkine_jacobe(b2k_chain_t chain, int dtype, const void *q, int64_t N, int64_t ldq,
                     const double *base, const double *tool, void *T, void *J, void *stream);

/* Planar forward kinematics and Jacobians of an ETS2 chain (reference ETS2.eval / fkine / jacob0 / jacobe, ET.py and
 * ETS.py; pure Python there).  The chain is created by b2k_chain_create from the ETS2's 3-D embedding (R -> Rz,
 * tx -> tx, ty -> ty, SE2 -> an SE3 acting in the xy plane); a chain with any other joint axis, or a constant with an
 * out-of-plane rotation or a z translation, is rejected before any CUDA call with an error naming the first such
 * transform.  base and tool are row-major 3x3 SE(2) matrices (NULL = identity); the base enters T only.
 *   T (N,3,3) row-major = base * prod_k ET2_k(q[i, jindex_k]) * tool
 *   J (N,3,n), rows (vx, vy, w), columns in chain order: frame 0 = jacob0, in the chain's start frame;
 *     frame 1 = jacobe = blkdiag(R^T, 1) jacob0, R the rotation of the pose (tool in, base out).
 * T or J may be NULL, not both; both from one pass when both are given.  n = 1..B2K_MAX_JOINTS, fp32 / fp64. */
int b2k_fkine_planar(b2k_chain_t chain, int dtype, const void *q, int64_t N, int64_t ldq, const double *base,
                     const double *tool, int frame, void *T, void *J, void *stream);

/* ---------------------------------------------------------------- inverse kinematics
 * Replaces fknm.IK_LM_c (fknm.cpp:394-525 -> _IK_LM_Chan/_Wampler/_Sugihara ik.cpp:157-209
 * -> _IK_loop ik.cpp:19-75) for N targets at once, and -- with semantics =
 * B2K_IK_SEM_PYTHON -- the Python solver behind ETS.ikine_LM (IK.py:297-367, 994-1017).
 *   Tep      (N,4,4) device, row-major
 *   q0       (N,n) device initial guesses or NULL (then drawn inside the joint limits)
 *   we       host 6-vector of Cartesian weights or NULL (= ones); We = diag(we)
 *   reject_jl  reject converged solutions outside the joint limits and restart
 *   seed     seed of the counter-based restart generator (the reference uses unseeded libc
 *            rand(), ik.cpp:293, or numpy default_rng, IK.py:166)
 *   rng_per_row  1: restart draws keyed by (seed,row,search); 0: shared by all rows
 *            (IKSolver.solve reuses one set of restarts for a whole trajectory, IK.py:222-272)
 * Outputs (device): q_out (N,n), success/iterations/searches int32 (N), residual (N) in dtype
 * -- the tuple IK_LM_c returns (fknm.cpp:516), one entry per target.
 * q0 and q_out hold the chain's n joints in chain order, i.e. q[ets.jindices] -- exactly what the reference's Python
 * solver hands back for an ETS whose jindices are not 0..n-1 (it pads q to max_jindex + 1 internally, IK.py:216-240,
 * and returns q[ets.jindices], IK.py:346), so sub-chains of a larger robot are served as they are (the reference's
 * C++ loop assumes dense jindices, ik.cpp:34-35).  Two joints sharing one jindex are rejected.
 * method = B2K_IK_NR / B2K_IK_GN select fknm.IK_NR_c / IK_GN_c (fknm.cpp:164-392) and, with the
 * Python semantics, IK_NR.step / IK_GN.step (IK.py:714-762, 1154-1219; both take pinv(J) e there).
 * The pseudo-inverse step is evaluated as Jw^T (Jw Jw^T + d^2)^-1 ew (6x6 Cholesky); pinv = False
 * on a square chain (J.inverse() e) is the same vector and is not a separate code path.
 */
int b2k_ik_lm(b2k_chain_t chain, int dtype, const void *Tep, int64_t N, const void *q0,
              int ilimit, int slimit, double tol, int reject_jl, const double *we, double lambda,
              int method, uint64_t seed, int semantics, int rng_per_row, void *q_out,
              int32_t *success, int32_t *iterations, int32_t *searches, void *residual,
              void *stream);

/* The Python solver loop of b2k_ik_lm (always B2K_IK_SEM_PYTHON) with the null-space terms of the reference's
 * IK_LM / IK_NR / IK_GN (IKSolver._calc_qnull / _null_Σ, IK.py), for redundant chains (7 <= n <= 10).  Arguments
 * as b2k_ik_lm, plus:
 *   kq   joint-limit avoidance gain; > 0 turns the term on (the reference's `if λΣ > 0`)
 *   km   manipulability gain; > 0 turns the term on
 *   ps   scalar; pi  host n-vector, the influence distance of each joint's limits
 * Every step, at the pre-step q and with the unweighted base-frame J:
 *   q <- q + dq_solver + qnull,  qnull = (I - pinv(J) J) g
 *   g = [kq > 0] sigma(q) / kq + [km > 0] jacobm(q) / km       (jacobm as b2k_jacobm with all six axes)
 *   sigma_i = +((q_i - l_i) - pi_i)^2 / (ps - pi_i)^2  if q_i - l_i <= pi_i
 *           = -((h_i - q_i) - pi_i)^2 / (ps - pi_i)^2  if h_i - q_i <= pi_i (wins when both hold); 0 otherwise
 * with l, h the chain's joint limits in chain order (a sub-chain of a larger robot uses its own joints, where the
 * reference indexes its padded q by position).  The projector is formed as g - J^T (J J^T)^-1 J g from the Cholesky
 * factor of J J^T; where that factor does not exist (J close to losing row rank) the search is abandoned, as a
 * singular step is.  Rejected before any CUDA call: everything b2k_ik_lm rejects, n < 7 (a full-rank J of n <= 6
 * joints has no null space: call b2k_ik_lm), non-finite kq, km, ps or pi, neither kq nor km > 0, and ps == pi[i]
 * with kq > 0 (the reference divides by zero there).
 */
int b2k_ikine_null(b2k_chain_t chain, int dtype, const void *Tep, int64_t N, const void *q0,
                   int ilimit, int slimit, double tol, int reject_jl, const double *we, double lambda,
                   int method, uint64_t seed, int rng_per_row, double kq, double km, double ps,
                   const double *pi, void *q_out, int32_t *success, int32_t *iterations,
                   int32_t *searches, void *residual, void *stream);

/* The Python solver loop of b2k_ik_lm (always B2K_IK_SEM_PYTHON) with the quadratic-programming step of the
 * reference's IK_QP (ETS.ikine_QP), for 1 <= n <= 10.  Arguments as b2k_ik_lm without lambda, method and semantics
 * (we weighs only the cost E), plus:
 *   kj, ks  joint-velocity and slack gains (> 0)
 *   kq      velocity-damper gain; > 0 turns the damper on
 *   km      manipulability gain; > 0 turns the term on (needs n >= 6)
 *   ps      scalar; pi  host n-vector, the influence distance of each joint's limits (read only when kq > 0)
 * Every step, at the pre-step q with the unweighted angle-axis error e and the base-frame J, dq is the exact minimiser of
 *   1/2 kj |dq|^2 + 1/2 w |s|^2 + c^T dq   subject to  J dq + s = e,   w = ks / sum|e|,  c = -[km > 0] jacobm(q) / km
 * (jacobm as b2k_jacobm with all six axes) and, when kq > 0, one damper row per joint within pi_i of a limit:
 *   -dq_i <= ((q_i - l_i) - ps) / ((pi_i - ps) kq)  if q_i - l_i <= pi_i
 *    dq_i <= ((h_i - q_i) - ps) / ((pi_i - ps) kq)  if h_i - q_i <= pi_i (this row wins when both hold)
 * with l, h the chain's joint limits in chain order; q <- q + dq.  A row with sum|e| = 0 steps by 0 (its E is 0).  A QP
 * whose factorisation fails or that is not solved within 2n + 2 active-set rounds abandons the search.  Rejected
 * before any CUDA call: what b2k_ik_lm rejects, non-finite kj, ks, kq, km or ps, kj <= 0 or ks <= 0, with kq > 0 a
 * NULL or non-finite pi or ps == pi[i], and km > 0 with n < 6 (J J^T is singular there).
 */
int b2k_ikine_qp(b2k_chain_t chain, int dtype, const void *Tep, int64_t N, const void *q0,
                 int ilimit, int slimit, double tol, int reject_jl, const double *we, uint64_t seed,
                 int rng_per_row, double kj, double ks, double kq, double km, double ps, const double *pi,
                 void *q_out, int32_t *success, int32_t *iterations, int32_t *searches, void *residual,
                 void *stream);

/* ---------------------------------------------------------------- inverse dynamics (DH RNE)
 * b2k_rne_create replaces frne.init (frne.c:233-299): n links, mdh = 0 standard / 1 modified
 * DH, L = 24 doubles per link packed as reference DHRobot.py:1340-1358
 *   [alpha, a, theta, d, sigma, offset, m, r(3), I(9 row-major), Jm, G, B, Tc+, Tc-].
 * b2k_rne replaces the per-row frne.frne loop (frne.c:106-230 -> newton_euler ne.c:62-492):
 *   tau[i] = RNE(q[i], qd[i], qdd[i]) for i < N, arrays (N,n).
 *   grav : host 3-vector handed to the recursion as the base acceleration, i.e. MINUS the
 *          robot's gravity exactly as DHRobot.rne passes it (DHRobot.py:1449); must not be NULL
 *   fext : host 6-vector wrench at the tip or NULL (= zeros)
 * q, qd, qdd need the alignment of their element type; tau is written in pieces of 16 bytes when a row of tau (n reals)
 * is a multiple of 16 bytes, else 8 when it is a multiple of 8, else 4, and must be aligned to that piece (an fp64
 * 6-joint tau: 16 bytes).  A misaligned or NULL (N > 0) array is rejected before any CUDA call.
 */
int b2k_rne_create(int n, int mdh, const double *L, b2k_rne_t *out);
int b2k_rne_destroy(b2k_rne_t rne);
int b2k_rne(b2k_rne_t rne, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
            const double *grav, const double *fext, void *tau, void *stream);
/* b2k_rne_wrench: b2k_rne plus the base wrench of every row (DHRobot.rne(..., base_wrench=True)).  tau is what
 * b2k_rne writes; wbase (N,6) device = [fx, fy, fz, mx, my, mz], the force and moment the base exerts on link 1,
 * expressed in frame 0 (the frame of grav), moment about the origin of frame 0.  The actuator terms (Jm, G, B, Tc) act
 * inside the joints and do not enter it; fext enters as it enters tau.  wbase must be 2*sizeof(real)-byte aligned.
 * Rejects what b2k_rne rejects plus a NULL (N > 0) or misaligned wbase, before any CUDA call. */
int b2k_rne_wrench(b2k_rne_t rne, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                   const double *grav, const double *fext, void *tau, void *wbase, void *stream);

/* Robot-specialised kernels.  For all-revolute arms b2k_rne (and the dynamics entry points below) run a kernel that is
 * generated for THIS robot's link table and compiled for sm_90a at first use (NVRTC): terms whose link parameter is zero
 * are never emitted, alpha = k pi/2 turns rotations into permutations, constants are folded (csrc/b2k_rne_gen.cpp,
 * b2k_rne_spec.cu).  Results equal the generic kernel's to rounding.  A modified-DH arm with a prismatic first joint has a
 * non-symmetric M under the kept reference treatment of that joint, which the specialised accel solve (pivot-free LDL^T)
 * cannot handle: its accel is served by the generic kernel, and b2k_rne_fdyn refuses it.  Environment: B2K_RNE_SPEC=0 disables it, =2 makes a
 * failure to specialise an error; B2K_NVRTC_PATH names libnvrtc.so.12 when it is not on the loader path.
 *   b2k_rne_spec_info  writes a one-line description of the kernel that serves (mode, dtype, grav pattern, has_fext) for
 *                      this robot into buf -- mode: 0 rne, 1 inertia, 2 gravload, 3 itorque, 4 coriolis, 5 accel,
 *                      6 rne with the base wrench (b2k_rne_wrench; codegen: n + 6 outputs, tau then wbase).
 *   b2k_rne_codegen    returns the generated row function (plain C in terms of `real`; also valid host C++) and its
 *                      constant bank, so the generator can be checked against the oracle without a GPU;
 *                      counts[3] = multiplications, fused multiply-adds, additions per row. */
int b2k_rne_spec_info(b2k_rne_t rne, int mode, int dtype, const double *grav, int has_fext, char *buf, int64_t cap);
int b2k_rne_codegen(b2k_rne_t rne, int mode, int grav_mask, int has_fext, char *src, int64_t src_cap, double *consts,
                    int32_t consts_cap, int32_t *n_consts, int32_t *counts);

/* ---------------------------------------------------------------- inverse dynamics of ETS / URDF robots (rigid-body trees)
 * Replaces the pure-Python Robot.rne (Robot.py:1704-1903: Featherstone's recursion over spatial vectors, one Python loop
 * iteration per trajectory row).  The tree is described the way that function walks it: n joint groups in link order;
 * group j hangs off group parent[j] (-1 = the base) through the constant transform C[j] (3x4 row-major: the static links
 * of the group and the constant part of the joint link, folded) followed by ONE joint of kind axis[j] (B2K_RX..B2K_TZ,
 * flip[j]) that reads q[jindex[j]]; I6[j] (6x6 row-major, [linear; angular] order as spatialmath's SpatialInertia) is the
 * inertia of the group in the joint link's frame.  b2k_tree_rne: tau (N,n) = rne(q, qd, qdd) rows, arrays (N,n) device,
 * 16-byte aligned; grav = MINUS the robot's gravity (Robot.rne's a_grav), host 3-vector.  Reference quirks kept: the
 * joint motion subspace ignores `flip` (ET.s, ET.py:592-608), torques are listed in group order.  The kernel is generated
 * for the tree at hand and compiled with NVRTC at first use (there is no pre-compiled kernel for an arbitrary tree). */
int b2k_tree_create(int n, const int32_t *parent, const int32_t *axis, const int32_t *flip, const int32_t *jindex,
                    const double *C, const double *I6, b2k_tree_t *out);
int b2k_tree_destroy(b2k_tree_t tree);
int b2k_tree_rne(b2k_tree_t tree, int dtype, const void *q, const void *qd, const void *qdd, int64_t N, const double *grav,
                 void *tau, void *stream);
/* The operations DynamicsMixin derives from rne (Dynamics.py: inertia 752-758, gravload 912-915, itorque 1456-1459,
 * coriolis 825-857, accel 490-503) for a tree robot -- in the reference n to n(n+1)/2 + 1 Python rne loops per row, here
 * one generated kernel per operation (the same recursion over symbolic unit / zero inputs, like the DH entry points below).
 *   op B2K_DYN_INERTIA  in0 = q                      out (N,n,n)  row i = rne(q, 0, e_i, gravity 0)
 *      B2K_DYN_GRAVLOAD in0 = q                      out (N,n)    rne(q, 0, 0)                          uses grav
 *      B2K_DYN_ITORQUE  in0 = q, in1 = qdd           out (N,n)    rne(q, 0, qdd, gravity 0)
 *      B2K_DYN_CORIOLIS in0 = q, in1 = qd            out (N,n,n)  the reference's combination rule
 *      B2K_DYN_ACCEL    in0 = q, in1 = qd, in2 = tau out (N,n)    M(q)^-1 (tau - rne(q, qd, 0))         uses grav
 * (B2K_DYN_RNE = b2k_tree_rne).  e_i and the input columns are in q order, the torque columns in group order, exactly as
 * the reference's calls produce them.  b2k_tree_codegen / b2k_tree_info take the same op codes. */
#define B2K_DYN_RNE 0
#define B2K_DYN_INERTIA 1
#define B2K_DYN_GRAVLOAD 2
#define B2K_DYN_ITORQUE 3
#define B2K_DYN_CORIOLIS 4
#define B2K_DYN_ACCEL 5
int b2k_tree_dyn(b2k_tree_t tree, int op, int dtype, const void *in0, const void *in1, const void *in2, int64_t N,
                 const double *grav, void *out, void *stream);
/* Exact first derivatives of the tree's dynamics (forward-mode tangents of the generated recursion, never differences),
 * for linearising about a batch of states (MPC, iLQR / DDP, LQR):
 *   op B2K_DYN_RNE_DERIV   x = qdd     out0 = dtau_dq (N,n,n), out1 = dtau_dqd (N,n,n); out2 must be NULL
 *      B2K_DYN_ACCEL_DERIV x = torque  out0 = dqdd_dq, out1 = dqdd_dqd, out2 = dqdd_dtau (N,n,n) each
 * Entry [i, k] = d out_i / d x_k: i in group order as b2k_tree_rne returns tau (op 7) or in the order of B2K_DYN_ACCEL's
 * output (op 8), k in q order.  Op 8 differentiates qdd* = accel(q, qd, torque) with accel's M and solve:
 * dqdd_dx = -M^-1 dtau_dx at qdd*, dqdd_dtau = M^-1.  grav = MINUS the robot's gravity, as for b2k_tree_rne.  Arrays are
 * device, 16-byte aligned.  b2k_tree_dyn rejects these two op codes; b2k_tree_codegen / b2k_tree_info take them (op 8
 * generates two functions: rne_row, the ACCEL row, and rne_deriv_row, the op 7 row evaluated at qdd*). */
#define B2K_DYN_RNE_DERIV 7
#define B2K_DYN_ACCEL_DERIV 8
int b2k_tree_derivatives(b2k_tree_t tree, int op, int dtype, const void *q, const void *qd, const void *x, int64_t N,
                         const double *grav, void *out0, void *out1, void *out2, void *stream);
/* The dynamics regressor of a tree, for identifying its inertial parameters from logged (q, qd, qdd, tau):
 * tau = Y(q, qd, qdd; g) pi exactly, for any rigid-body group inertia.  pi has p = 10 n entries, 10 per joint group in
 * group order (the order of b2k_tree_rne's tau):  pi[10j .. 10j+9] = [m, hx, hy, hz, Ixx, Iyy, Izz, Ixy, Iyz, Ixz]
 * with I6[j] = [[m E, -[h]x], [[h]x, Ib]], Ib = [[Ixx, Ixy, Ixz], [Ixy, Iyy, Iyz], [Ixz, Iyz, Izz]] (for point masses
 * h = sum m r, Ib = sum m (r.r E - r r^T)).  Y[i, 10k .. 10k+9] is exact 0 unless group k is group i or hangs below it.
 * Y does not depend on I6.  There are no friction or motor columns: b2k_tree_rne has no such terms.
 *   b2k_tree_regressor       Y (N, n, 10n) row-major, one launch of a kernel generated for the tree (NVRTC, op code
 *                            B2K_DYN_REGRESSOR); grav = MINUS the robot's gravity, as for b2k_tree_rne.  q, qd, qdd, Y
 *                            device, 16-byte aligned.
 *   b2k_tree_regressor_gram  the normal equations, always in fp64, without Y existing in full: G (p, p) = sum Y^T W Y,
 *                            b (p) = sum Y^T W tau, s (1) = sum tau^T W tau, W = diag(weights) (host, n values in group
 *                            order, finite and >= 0; NULL = all 1).  tau (N, n) has the compute type and group order.
 *                            G is exactly symmetric and equal calls give equal bits.  G, b, s are device arrays, 8-byte
 *                            aligned, written also for N = 0 (zeros, no kernel).
 * b2k_tree_dyn and b2k_tree_derivatives reject B2K_DYN_REGRESSOR; b2k_tree_codegen / b2k_tree_info take it (the generated
 * function, rne_regressor_row(..., i, y), writes joint row i of Y).  Every argument is checked before any CUDA call. */
#define B2K_DYN_REGRESSOR 10
int b2k_tree_regressor(b2k_tree_t tree, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                       const double *grav, void *Y, void *stream);
int b2k_tree_regressor_gram(b2k_tree_t tree, int dtype, const void *q, const void *qd, const void *qdd, const void *tau,
                            int64_t N, const double *grav, const double *weights, double *G, double *b, double *s,
                            void *stream);
int b2k_tree_codegen(b2k_tree_t tree, int op, int grav_mask, char *src, int64_t src_cap, double *consts, int32_t consts_cap,
                     int32_t *n_consts, int32_t *counts);
int b2k_tree_info(b2k_tree_t tree, int op, int dtype, const double *grav, char *buf, int64_t cap);

/* ---------------------------------------------------------------- dynamics built on the recursion
 * The reference's DynamicsMixin (robot/Dynamics.py) obtains these by looping frne calls in
 * Python; here each is ONE kernel in which a lane performs all the recursions of its row
 * (SURVEY 8f-1).  q, qd, qdd, torque are (N,n) device arrays; gravity conventions as b2k_rne
 * (grav = MINUS the robot's gravity, host 3-vector).
 *   b2k_rne_inertia   M (N,n,n): row i of M[k] = rne(q_k, 0, e_i, g=0)          Dynamics.py:704-763
 *   b2k_rne_gravload  taug (N,n) = rne(q, 0, 0, g)                              Dynamics.py:863-921
 *   b2k_rne_itorque   taui (N,n) = rne(q, 0, qdd, g=0)                          Dynamics.py:1407-1465
 *   b2k_rne_coriolis  C (N,n,n), on a friction-free copy of the robot           Dynamics.py:765-861
 *   b2k_rne_accel     qdd (N,n) = M^-1 (torque - rne(q, qd, 0, g)), friction kept  Dynamics.py:424-510
 *   b2k_rne_derivatives        dtau_dq, dtau_dqd (N,n,n), [i,k] = d tau_i / d x_k of tau = rne(q, qd, qdd, g, fext)
 *                              (viscous friction adds G^2 B to the diagonal of dtau_dqd, Coulomb friction adds 0)
 *   b2k_rne_accel_derivatives  at qdd* = b2k_rne_accel(q, qd, torque, g), with M = b2k_rne_inertia(q):
 *                              dqdd_dq = -M^-1 dtau_dq, dqdd_dqd = -M^-1 dtau_dqd (both at qdd*), dqdd_dtau = M^-1
 *   (no reference counterpart: exact forward-mode tangents of the recursion, one launch each; fext may be NULL)
 * Inputs need the alignment of their element type.  The output is written in pieces of 16 bytes when one of its rows (n
 * or n*n reals) is a multiple of 16 bytes, else 8 when it is a multiple of 8, else 4, and must be aligned to that piece;
 * a misaligned or NULL (N > 0) array is rejected before any CUDA call.
 */
int b2k_rne_inertia(b2k_rne_t rne, int dtype, const void *q, int64_t N, void *M, void *stream);
int b2k_rne_gravload(b2k_rne_t rne, int dtype, const void *q, int64_t N, const double *grav, void *taug, void *stream);
int b2k_rne_itorque(b2k_rne_t rne, int dtype, const void *q, const void *qdd, int64_t N, void *taui, void *stream);
int b2k_rne_coriolis(b2k_rne_t rne, int dtype, const void *q, const void *qd, int64_t N, void *C, void *stream);
int b2k_rne_accel(b2k_rne_t rne, int dtype, const void *q, const void *qd, const void *torque, int64_t N,
                  const double *grav, void *qdd, void *stream);
int b2k_rne_derivatives(b2k_rne_t rne, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                        const double *grav, const double *fext, void *dtau_dq, void *dtau_dqd, void *stream);
int b2k_rne_accel_derivatives(b2k_rne_t rne, int dtype, const void *q, const void *qd, const void *torque, int64_t N,
                              const double *grav, void *dqdd_dq, void *dqdd_dqd, void *dqdd_dtau, void *stream);

/* The dynamics regressor, for identifying a DH arm's link parameters from logged (q, qd, qdd, tau):
 * tau = Y(q, qd, qdd; g) pi with no tip wrench, for every link table rne serves (prismatic joints through d = q + offset,
 * the modified-DH prismatic first joint as rne treats it, flip ignored).  pi has p = 14 n entries, link-major, 14 per
 * link j:  pi[14j .. 14j+13] = [m, m rx, m ry, m rz, Ixx, Iyy, Izz, Ixy, Iyz, Ixz, Jm, B, Tc+, Tc-]
 * r is the link's centre of mass in its frame (as rne takes it); the six inertia entries, in the order of the 6-vector
 * form of a link's I, are those of I_o = I + m (r.r E - r r^T), the inertia about the link-frame origin.  The gear ratio
 * G is a known constant: the columns of Jm_j, B_j, Tc+_j, Tc-_j are G_j^2 qdd_j, G_j^2 qd_j, |G_j| [qd_j > 0],
 * |G_j| [qd_j < 0] in row j and 0 elsewhere; Y[j, 14i + k] = 0 for i < j.  These zeros are written as exact 0.
 *   b2k_rne_regressor       Y (N, n, 14n) row-major, one launch; grav = MINUS the robot's gravity, as b2k_rne.
 *                           The arrays follow the rules above (Y's row is 14 n^2 reals).
 *   b2k_rne_regressor_gram  the normal equations without Y existing in full, always in fp64:
 *                           G (p, p) = sum Y^T W Y, b (p) = sum Y^T W tau, s (1) = sum tau^T W tau over the N rows,
 *                           W = diag(weights) (host, n values, finite and >= 0; NULL = all 1).  tau (N, n) has the
 *                           compute type.  G is exactly symmetric, and no atomics are used: equal calls give equal bits.
 *                           G, b, s are device arrays, 8-byte aligned, written also for N = 0 (zeros, no kernel).
 * Every argument is checked before any CUDA call.  No reference counterpart. */
int b2k_rne_regressor(b2k_rne_t rne, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                      const double *grav, void *Y, void *stream);
int b2k_rne_regressor_gram(b2k_rne_t rne, int dtype, const void *q, const void *qd, const void *qdd, const void *tau,
                           int64_t N, const double *grav, const double *weights, double *G, double *b, double *s,
                           void *stream);

/* ---------------------------------------------------------------- static forces (DynamicsMixin, robot/Dynamics.py)
 * One forward walk over a compiled chain per row (base and tool as the chain has them, as for b2k_jacob0); q is (N, ldq)
 * with the joint coordinates at the chain's joint indices.  Unlike b2k_rne, `grav` is the world-frame gravity AS THE
 * ROBOT STORES IT (host 3-vector, not negated).  `mass` is a host table of n x 4 doubles (m_j, c_j): c_j is link j's
 * centre of mass in the frame right after joint j's elementary transform.  Flipped joints follow the chain, as in
 * b2k_jacob0 (b2k_rne ignores flip).  Wrenches W = [fx fy fz mx my mz] are device arrays: w_stride 0 = one wrench for
 * every row, 6 = (N, 6).  frame 0: W in the world frame; 1: in the end-effector frame.  b2k_pay_jacobian and
 * b2k_friction check their arguments as the chain entry points do (n range instead of a chain; device arrays aligned to
 * their element size).
 *   b2k_gravjac      taug (N,n) = -sum_i J_ci^T m_i g and J0 (N,6,n) = jacob0       DynamicsMixin.gravjac
 *   b2k_pay          tau (N,n) = -J^T W, J = jacob0 (frame 0) or jacobe (frame 1)  DynamicsMixin.pay (given q)
 *   b2k_pay_jacobian tau (N,n) = -J^T W from a given J (N,6,n)                      DynamicsMixin.pay (given J)
 *   b2k_paycap       wmax (N,n), joint (N) int32: with w^ = w / |w| per row, tau_B the gravity load and
 *                    tau_P = pay(w^), wmax_j = (tauR[j,0] - tau_B,j) / tau_P,j if tau_P,j > 0, (tauR[j,1] - tau_B,j) /
 *                    tau_P,j if < 0, +inf if 0; joint = first argmin; a zero w row gives NaN and -1.
 *                    tauR: host n x 2 doubles (max, min)                              DynamicsMixin.paycap
 *   b2k_friction     tau (N,n) = -(G^2 B qd + |G| Tc(qd)), Tc(qd) = Tc+ (qd > 0), Tc- (qd < 0), 0;
 *                    params: host n x 4 doubles (B, G, Tc+, Tc-)                      Link.friction / DynamicsMixin.friction
 */
int b2k_gravjac(b2k_chain_t chain, int dtype, const void *q, int64_t N, int64_t ldq, const double *mass, const double *grav,
                void *taug, void *J0, void *stream);
int b2k_pay(b2k_chain_t chain, int dtype, const void *q, int64_t N, int64_t ldq, const void *W, int64_t w_stride, int frame,
            void *tau, void *stream);
int b2k_pay_jacobian(int dtype, int n, const void *J, const void *W, int64_t w_stride, int64_t N, void *tau, void *stream);
int b2k_paycap(b2k_chain_t chain, int dtype, const void *q, int64_t N, int64_t ldq, const double *mass, const double *grav,
               const void *w, int64_t w_stride, int frame, const double *tauR, void *wmax, int32_t *joint, void *stream);
int b2k_friction(int dtype, int n, const double *params, const void *qd, int64_t N, void *tau, void *stream);

/* b2k_rne_fdyn integrates the forward dynamics of an ENSEMBLE of initial states (DynamicsMixin.fdyn, Dynamics.py:185-422,
 * integrates one): one lane per trajectory, Dormand-Prince 5(4) with scipy RK45's step control (rtol, atol, max_step,
 * first_step <= 0: automatic), every stage's acceleration from the robot-specialised recursion.  q0, qd0 (ntraj,n) device
 * (qd0 may be NULL = at rest).  Torque: torque_mode 0 none, 1 constant tau (host n), 2 tau_rows (ntraj,n) device,
 * 3 PD kp (qstar - q) - kd qd (host n-vectors).  Output, M slots per trajectory: grid = 0 the accepted steps (t, q, qd as
 * scipy's integrator visits them), grid = 1 the uniform grid k dt by linear interpolation (the reference's interp1d);
 * out_t (ntraj,M), out_q / out_qd (ntraj,M,n), out_count (samples produced; > M means the capacity was too small),
 * out_status (bit 0: step size underflow, bit 1: capacity exceeded).  All-revolute robots; needs NVRTC. */
int b2k_rne_fdyn(b2k_rne_t rne, int dtype, const void *q0, const void *qd0, int64_t ntraj, double T, const double *grav,
                 int torque_mode, const double *tau, const void *tau_rows, const double *kp, const double *kd, const double *qstar,
                 double rtol, double atol, double max_step, double first_step, double dt, int grid, int M, void *out_t,
                 void *out_q, void *out_qd, int32_t *out_count, int32_t *out_status, void *stream);
/* the same integrator around the accel recursion of a rigid-body tree (Robot.fdyn); grav = MINUS the robot's gravity */
int b2k_tree_fdyn(b2k_tree_t tree, int dtype, const void *q0, const void *qd0, int64_t ntraj, double T, const double *grav,
                 int torque_mode, const double *tau, const void *tau_rows, const double *kp, const double *kd, const double *qstar,
                 double rtol, double atol, double max_step, double first_step, double dt, int grid, int M, void *out_t,
                 void *out_q, void *out_qd, int32_t *out_count, int32_t *out_status, void *stream);

/* Fixed-step rollouts with discrete-time sensitivities, for sampling MPC and shooting methods (iLQR / DDP): one lane per
 * trajectory, K classical RK4 steps of x = [q; qd] under a torque held over each step,
 *   f(x, tau) = [qd; accel(q, qd, tau)]     k1 = f(x_k), k2 = f(x_k + dt/2 k1), k3 = f(x_k + dt/2 k2), k4 = f(x_k + dt k3)
 *   x_{k+1} = x_k + dt/6 (k1 + 2 k2 + 2 k3 + k4)
 * with accel exactly that of the robot (b2k_rne_accel: friction and armature kept; b2k_tree_dyn B2K_DYN_ACCEL).  A (N,K,2n,2n)
 * and B (N,K,2n,n) are the exact derivatives of that map, A_k = d x_{k+1} / d x_k and B_k = d x_{k+1} / d tau_k, [i, j] =
 * d out_i / d in_j, chained through the four stages from the derivatives of accel at each stage state (Coulomb friction
 * contributes 0).  A singular M gives non-finite values from that step on; no error is raised.
 *   q0, qd0 (N,n) device (qd0 may be NULL = at rest); tau (K,n) device with tau_stride 0 (one sequence for every trajectory)
 *   or (N,K,n) with tau_stride K n; q, qd (N,K+1,n) device, index 0 the initial state.  A and B both NULL: states only;
 *   both non-NULL: with sensitivities (the states are bit-identical either way); one NULL is rejected.  Every array needs
 *   the alignment of its element type.  dt finite and > 0, K >= 1, grav as the family's accel takes it (MINUS the robot's
 *   gravity).  DH arms must be all-revolute.  Every argument is checked, and the kernel built (NVRTC), before any CUDA
 *   call; N = 0 launches nothing.  b2k_rne_spec_info / b2k_tree_info describe the kernels with mode / op 305 (states only)
 *   and 308 (with sensitivities). */
int b2k_rne_rollout(b2k_rne_t rne, int dtype, const void *q0, const void *qd0, int64_t N, int32_t K, double dt,
                    const double *grav, const void *tau, int64_t tau_stride, void *q, void *qd, void *A, void *B, void *stream);
int b2k_tree_rollout(b2k_tree_t tree, int dtype, const void *q0, const void *qd0, int64_t N, int32_t K, double dt,
                     const double *grav, const void *tau, int64_t tau_stride, void *q, void *qd, void *A, void *B, void *stream);

/* ---------------------------------------------------------------- operational-space dynamics
 * The arithmetic of DynamicsMixin.inertia_x, coriolis_x, gravload_x and accel_x (robot/Dynamics.py, between gravload and
 * itorque: per row np.linalg.inv / pinv of the analytical Jacobian and numpy triple products, in a Python loop), as an
 * epilogue over what the joint-space entry points produced.  All arrays are (N, ...) device arrays of dtype, row-major:
 *   Ja (N,6,n) analytical Jacobian (b2k_jacob0_analytical)   Ji_in (N,n,6) a given inverse (then Ja is not inverted)
 *   M, C (N,n,n) inertia / Coriolis matrix    Jd (N,6,n) time derivative of Ja    G (N,n) gravity load
 *   Mx_in (N,6,6) a given Mx (Cx then needs no M)    xd (N,6) task-space velocity    w (N,6) wrench
 * inverse B2K_OPS_INV: Ji = inv(Ja), n must be 6, partial pivoting as LAPACK getrf; a row with an exactly zero pivot gets
 * NaN in every output that depends on Ji (numpy raises LinAlgError for it).  B2K_OPS_PINV: Ji = pinv(Ja) by one-sided
 * Jacobi SVD, singular values <= 1e-15 s_max dropped as numpy.linalg.pinv does.  The cut is the same in fp32, where it
 * keeps a singular value that is zero in exact arithmetic but ~1e-8 s_max after rounding, so the fp32 pseudo-inverse of
 * a numerically rank-deficient Ja is not meaningful; only exact structure is dropped reliably (an all-zero column of Ja
 * for n <= 6, an all-zero row for n >= 7).  One launch writes any non-NULL output:
 *   Ji  (N,n,6)                                                         needs Ja or Ji_in
 *   Mx  (N,6,6) = Ji^T M Ji                      (inertia_x)            needs M
 *   Cx  (N,6,6) = Ji^T C Ji - Mx Jd Ji           (coriolis_x)           needs C, Jd and M or Mx_in
 *   Gx  (N,6)   = Ji^T G                         (gravload_x)           needs G
 *   qd  (N,n)   = Ji xd                          (accel_x, first stage) needs xd
 *   tau (N,n)   = Ja^T w                         (accel_x, first stage) needs Ja and w
 * b2k_opspace_xdd is the last stage of accel_x: xdd (N,6) = Ja qdd + Jd qd, with qdd from b2k_rne_accel / b2k_tree_dyn
 * and Jd taken at qd.  Arguments are validated before any CUDA call. */
#define B2K_OPS_INV 0
#define B2K_OPS_PINV 1
int b2k_opspace(int dtype, int n, int inverse, const void *Ja, const void *Ji_in, const void *M, const void *C, const void *Jd,
                const void *G, const void *Mx_in, const void *xd, const void *w, int64_t N, void *Ji, void *Mx, void *Cx, void *Gx,
                void *qd, void *tau, void *stream);
int b2k_opspace_xdd(int dtype, int n, const void *Ja, const void *qdd, const void *Jd, const void *qd, int64_t N, void *xdd,
                    void *stream);

/* ---------------------------------------------------------------- closed-form inverse kinematics
 * b2k_ikine_6s replaces DHRobot.ikine_6s (robot/DHRobot.py), which Puma560.ikine_a calls: the analytic joint solution of a
 * wrist-partitioned standard-DH 6R arm with the Puma link pattern, one pose per row, no iteration.
 *   dh   host (6,4) rows of (d, a, alpha, offset).  The pattern, each condition to 1e-9: alpha = (+pi/2, 0, -pi/2, s pi/2,
 *        -s pi/2, any) with s = +1 or -1, a1 = a4 = a5 = 0, d5 = 0, a2 != 0.  Anything else is B2K_ERR_INVALID.
 *   base, tool  host 4x4 row-major, NULL = identity
 *   T    (N,4,4) device poses of dtype
 *   conf host array of nconf (1..8) configuration codes: bit 0 set = shoulder right ("r", else "l"), bit 1 set = elbow
 *        down ("d", else "u"), bit 2 set = wrist flipped ("f", else "n")
 *   q    (N,nconf,6) joint angles wrapped into [-pi, pi), the solution for conf[k] in slot k; NaN where out of reach
 *   ok   (N,nconf) int32: 1 = solved, 0 = the pose is out of reach for that configuration
 * Joint limits are not applied (the reference does not apply them either).  One launch; arguments are validated before
 * any CUDA call, and N = 0 returns without touching the device. */
int b2k_ikine_6s(int dtype, const double *dh, const double *base, const double *tool, const void *T, int64_t N, int nconf,
                 const int32_t *conf, void *q, int32_t *ok, void *stream);
/* b2k_ikine_ur is the same for UR-type arms (DHRobot.ikine_ur; the reference has no counterpart): the analytic joint
 * solution of a standard-DH 6R arm whose axes 2, 3 and 4 are parallel, one pose per row, no iteration.
 *   dh   the pattern, each condition to 1e-9: alpha = (+pi/2, 0, 0, +pi/2, -pi/2, any), a1 = a4 = a5 = 0, a2 != 0,
 *        a3 != 0.  d2, d3 and d4 enter only through their sum.  Anything else is B2K_ERR_INVALID.
 *   conf bit 0 set = shoulder right ("r": O5 . x1 >= 0), bit 1 set = elbow down ("d"; "u" = the elbow above the
 *        shoulder-O4 line, base z up), bit 2 set = wrist flipped ("f"; "n" = sin(theta5) >= 0)
 *   base, tool, T, q, ok, the validation and the N = 0 rule as for b2k_ikine_6s.  A row is out of reach when its O5 is
 *        nearer the first axis than |d2 + d3 + d4| or when the elbow cosine exceeds 1 by more than 64 eps of dtype. */
int b2k_ikine_ur(int dtype, const double *dh, const double *base, const double *tool, const void *T, int64_t N, int nconf,
                 const int32_t *conf, void *q, int32_t *ok, void *stream);
/* b2k_ikine_panda is the same for Panda-type 7R arms at a given q7 (DHRobot.ikine_panda; the reference has no
 * counterpart): the analytic joint solution of a modified-DH 7R arm with joint 7's coordinate fixed per row, no iteration.
 *   dh   host (7,4) rows of (d, a, alpha, offset), link k = Rx(alpha_k) Tx(a_k) Rz(q_k + offset_k) Tz(d_k).  The pattern,
 *        each condition to 1e-9: alpha2 .. alpha6 = (-pi/2, +pi/2, +pi/2, -pi/2, +pi/2), a2 = a3 = a6 = 0,
 *        d2 = d4 = d6 = 0, hypot(a4, d3) != 0, hypot(a5, d5) != 0 (PandaMDH).  Anything else is B2K_ERR_INVALID.
 *   q7   (N,) device array of dtype, aligned to its element size, non-NULL when N > 0: q[.., 6] of every solution of
 *        the row, as given.  A non-finite q7 gives a NaN row with ok = 0.
 *   conf bit 0 set = shoulder right ("r": sin(theta2) >= 0), bit 1 set = elbow down ("d"; "u" = ((O2 - O4) x
 *        (O6 - O4)) . z4 >= 0), bit 2 set = wrist flipped ("f"; "n" = (O2 - O6) . x5 >= 0)
 *   q    (N,nconf,7) joints 1..6 wrapped into [-pi, pi) and q7; NaN where out of reach
 *   base, tool, T, ok, the validation and the N = 0 rule as for b2k_ikine_6s.  A row is out of reach when the elbow
 *        cosine exceeds 1 by more than 64 eps of dtype, or when the wrist needs |p| > h + 64 eps |O6 - O2| (DESIGN f-17). */
int b2k_ikine_panda(int dtype, const double *dh, const double *base, const double *tool, const void *T, const void *q7,
                    int64_t N, int nconf, const int32_t *conf, void *q, int32_t *ok, void *stream);

/* ---------------------------------------------------------------- pure functions of the Jacobian
 * The six functions below take a batch of Jacobians J (N,6,n), n = 1..B2K_MAX_JOINTS.  J, qd and the output must be
 * aligned to their element size.  Every argument is checked before any CUDA call; N = 0 needs no arrays (NULL is
 * accepted) and touches no device.
 * b2k_hessian replaces fknm.ETS_hessian0 / ETS_hessiane (fknm.cpp:583-783 -> _ETS_hessian
 * methods.cpp:16-32): H (N,n,6,n) from J (N,6,n); pass jacob0 for hessian0, jacobe for hessiane.
 * b2k_manipulability is the Yoshikawa measure of ETS.manipulability (ETS.py:1780-1787):
 * m = sqrt|det(Ja Ja^T)| over the Cartesian rows selected by axes_mask (bit k = row k of J;
 * 63 = all, 7 = translational, 56 = rotational); |det Ja| when Ja is square. */
int b2k_hessian(int dtype, int n, const void *J, int64_t N, void *H, void *stream);
/* b2k_partial_fkine: the order-th partial derivative of forward kinematics of ETS.partial_fkine0 (Haviland & Corke,
 * "Manipulator Differential Kinematics Part II"), D (N, n^(order-1), 6, n) from jacob0 J (N,6,n), order = 3..5:
 * D[a_1, ..., a_{order-1}, :, j] = d^(order-1) J[:, j] / dq_{a_1} ... dq_{a_{order-1}}, symmetric in the a's.  Order 1
 * is J itself and order 2 the Hessian of b2k_hessian.  J's columns are taken in chain order, as b2k_hessian takes
 * them. */
int b2k_partial_fkine(int dtype, int n, int order, const void *J, int64_t N, void *D, void *stream);
int b2k_manipulability(int dtype, int n, const void *J, int64_t N, uint32_t axes_mask, void *m, void *stream);
/* The singular-value measures of ETS.manipulability (ETS.py:1789-1796) over the Cartesian rows in axes_mask:
 * kind 0 "minsingular" = numpy svd(Ja)[-1] (the smallest of min(rows, n) singular values), kind 1 "invcondition" =
 * 1 / numpy.linalg.cond(Ja) = s_min / s_max.  One-sided Jacobi SVD per row, in registers / local memory. */
int b2k_manipulability_svd(int dtype, int n, const void *J, int64_t N, uint32_t axes_mask, int kind, void *m, void *stream);
/* b2k_jacob_dot: Jd (N,6,n) = sum_i H[i] qd[i], the Jacobian time derivative of Robot.jacob0_dot
 * (Robot.py:964-1099, representation None: np.tensordot(hessian0, qd, (0,0))), from J (N,6,n) and qd (N,n)
 * without materialising the Hessian.
 * b2k_jacobm: the manipulability Jacobian dm/dq (N,n) of ETS.jacobm (ETS.py:1628-1685) / Robot.jacobm
 * (Robot.py:1124-1232) over the Cartesian rows in axes_mask: Jm[i] = m * vec(Ja Ha_i^T) . vec(inv(Ja Ja^T)). */
int b2k_jacob_dot(int dtype, int n, const void *J, const void *qd, int64_t N, void *Jd, void *stream);
int b2k_jacobm(int dtype, int n, const void *J, int64_t N, uint32_t axes_mask, void *Jm, void *stream);

/* ---------------------------------------------------------------- pose error, position-based servo, trajectories
 * The eight functions below check every argument before any CUDA call.  Their device arrays must be aligned to their
 * element size (arrived: 4 bytes).  N = 0 needs no device arrays (NULL is accepted) and touches no device; an array
 * documented as optional may be NULL at any N.  Host tables that are not optional must not be NULL, whatever N is.
 * b2k_angle_axis replaces fknm.Angle_Axis (fknm.cpp:112-162 -> _angle_axis ik.cpp:241-286), batched:
 * e (N,6) = [translation error; angle-axis rotation error] between Te (N,4,4) and Tep.
 * tep_stride = 16: one target per row, Tep (N,4,4); tep_stride = 0: a single (4,4) target for every row.
 * b2k_p_servo is tools/p_servo.py:46-106 with method="angle-axis": v (N,6) = gain .* e (gain: host
 * 6-vector or NULL = ones), arrived (N) int32 = sum|e| < threshold. */
int b2k_angle_axis(int dtype, const void *Te, const void *Tep, int64_t N, int64_t tep_stride, void *e, void *stream);
int b2k_p_servo(int dtype, const void *Te, const void *Tep, int64_t N, int64_t tep_stride, const double *gain,
                double threshold, void *v, int32_t *arrived, void *stream);

/* b2k_p_servo_rpy is tools/p_servo.py:46-106 with the reference's default method="rpy": the error is taken in the
 * end-effector frame, e = [t(Te^-1 Tep); tr2rpy(Te^-1 Tep, order="zyx")]; arguments as b2k_p_servo.
 * b2k_jacob0_analytical is ETS.jacob0_analytical (ETS.py:1570-1626): Ja (N,6,n) = blkdiag(I, A^-1(Gamma(R))) J0 from
 * the poses T (N,4,4) and base-frame Jacobians J (N,6,n); representation 0 "rpy/xyz", 1 "rpy/zyx", 2 "eul", 3 "exp".
 * tr2rpy / tr2eul / rotvelxform belong to spatialmath-python (not under the reference tree): their documented
 * conventions are restated in csrc/b2k_pose.cu and pinned by derivative identities in tests/, not by the package. */
int b2k_p_servo_rpy(int dtype, const void *Te, const void *Tep, int64_t N, int64_t tep_stride, const double *gain,
                    double threshold, void *v, int32_t *arrived, void *stream);
int b2k_jacob0_analytical(int dtype, int n, const void *T, const void *J, int64_t N, int representation, void *Ja,
                          void *stream);

/* b2k_jtraj replaces tools.trajectory.jtraj (tools/trajectory.py:686-780): quintic joint-space blend
 * from q0 to qf (host n-vectors; qd0 / qd1 boundary velocities or NULL = 0) sampled at N points,
 * written straight into device buffers q, qd, qdd (N,n) (qd / qdd may be NULL) so the batch can feed
 * b2k_fkine / b2k_rne without touching the host.
 *   t == NULL: N samples of normalised time np.linspace(0, 1, N), tscal must be 1 (the `t: int` form);
 *   t != NULL: device vector of N sample times (dtype), tscal = max(t) (the time-vector form). */
int b2k_jtraj(int dtype, int n, const double *q0, const double *qf, const double *qd0, const double *qd1,
              int64_t N, const void *t, double tscal, void *q, void *qd, void *qdd, void *stream);

/* b2k_mtraj replaces tools.trajectory.quintic (trajectory.py:271-416), trapezoidal (429-615) and their
 * multi-axis form mtraj (617-684): n axes, each following a quintic (kind 0; boundary velocities qd0 / qdf
 * or NULL = 0) or trapezoidal (kind 1; V = per-axis velocity of the linear segment, NULL or NaN = the
 * reference's default 1.5 (qf - q0) / tf) profile from q0[j] to qf[j]; outputs s, sd, sdd (N,n) device
 * (sd / sdd may be NULL).  t == NULL: sample times 0, 1, ..., N-1 (the `t: int` form, tf must be N-1);
 * t != NULL: device vector of N sample times, tf = max(t).  tblend (host, n doubles or NULL) receives the
 * blend times of the trapezoidal profile.  "V too small" / "V too big" (trajectory.py:555-558) -> B2K_ERR_INVALID. */
int b2k_mtraj(int dtype, int kind, int n, const double *q0, const double *qf, const double *qd0, const double *qdf,
              const double *V, int64_t N, const void *t, double tf, void *s, void *sd, void *sdd, double *tblend,
              void *stream);

/* b2k_ctraj replaces tools.trajectory.ctraj (trajectory.py:782-841 -> SE3.interp): N poses between T0 and T1 (host,
 * 4x4 row-major) at the path fractions s (device, N values in [0,1], clipped): translation interpolated linearly,
 * orientation by unit-quaternion slerp along the shorter arc; T (N,4,4) device.
 * b2k_mstraj evaluates the sample table of tools.trajectory.mstraj (trajectory.py:852-1152): the caller plans the
 * segments on the host exactly as the reference does and passes the pieces in row order -- kind 0: quintic blend
 * (jtraj coefficients A B C E F per axis in coef[piece][axis][0..4], sampled at t = (k+1) dt over a blend of length
 * tscal), kind 1: linear segment (coef = q_prev, q_next; s = (t0 + k dt) / tscal) -- and q (N,n) is written on the device. */
int b2k_ctraj(int dtype, const double *T0, const double *T1, const void *s, int64_t N, void *T, void *stream);
int b2k_mstraj(int dtype, int n, int npieces, const int64_t *row0, const int64_t *rows, const int32_t *kind,
               const double *tscal, const double *t0, const double *dt, const double *coef, int64_t N, void *q, void *stream);

/* ---------------------------------------------------------------- host-buffer front ends
 * The same operations for callers that hold HOST arrays (what the reference's API takes):
 * the library streams row chunks host->device, runs the kernel and streams results back on
 * several CUDA streams so copies overlap compute.  Pinned host memory (b2k_host_alloc, or
 * memory the caller registered) gets full PCIe/C2C bandwidth; pageable memory works too.
 * Synchronous: results are complete in the host arrays on return.  device = CUDA ordinal.
 */
int b2k_host_alloc(void **ptr, int64_t bytes);
int b2k_host_free(void *ptr);
int b2k_fkine_jacob0_host(b2k_chain_t chain, int dtype, const void *q_host, int64_t N,
                          int64_t ldq, const double *base, const double *tool, void *T_host,
                          void *J_host, int device);
int b2k_fkine_host(b2k_chain_t chain, int dtype, const void *q_host, int64_t N, int64_t ldq,
                   const double *base, const double *tool, void *T_host, int device);
int b2k_rne_host(b2k_rne_t rne, int dtype, const void *q_host, const void *qd_host,
                 const void *qdd_host, int64_t N, const double *grav, const double *fext,
                 void *tau_host, int device);
/* the host-buffer form of b2k_rne_wrench: tau_host (N,n) and wbase_host (N,6) */
int b2k_rne_wrench_host(b2k_rne_t rne, int dtype, const void *q_host, const void *qd_host,
                        const void *qdd_host, int64_t N, const double *grav, const double *fext,
                        void *tau_host, void *wbase_host, int device);

/* number of kernel launches this library has issued in the calling process (all threads);
 * bench.py reports the delta over its timed region as "gpu_launches". */
int64_t b2k_launch_count(void);

/* Test hook: evaluates the kernels' in-house sincos (csrc/b2k_trig.cuh) on n device values so
 * its accuracy can be checked in isolation: s[i], c[i] = sin(x[i]), cos(x[i]). */
int b2k_selftest_sincos(int dtype, const void *x, int64_t n, void *s, void *c, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* B2KIN_H */
