// b2k_frames.cu -- the pose of several frames along ONE chain from a single walk: the device side of fkine_all
// (reference Robot.fkine_all, Robot.py:638-700; DHRobot.fkine_all, DHRobot.py:1018-1064 -- a Python loop over the
// links that multiplies link transforms one configuration at a time).
//
// A frame is "the pose right after joint `after` of the chain, times a constant tail" (the constant transforms of the
// link that follow its joint), or an absolute constant (`after` = -1: the base frame, links ahead of the first joint).
// One lane walks one configuration, T = base A_0 J_0(q) A_1 J_1(q) ..., entirely in registers; whenever the walk has
// passed the joint a frame hangs on, the lane forms T * tail and stores the 16 reals of the frame with 128-bit
// vector stores into row-major (N, slots, 4, 4) memory -- a row's frames are contiguous, a warp writes
// 32 x slots x 128 B (fp64) of consecutive memory.  The earlier form was one pose launch per frame over prefix chains
// (q re-read and the prefix re-walked per frame, frame-major output).
// HBM-bound: 16 reals per frame per row out, n reals per row in.
#include "b2k_fkj.cuh"

#define B2K_MAX_FRAMES 16 /* per launch; the host splits longer lists (each launch walks the chain again) */

template <typename real>
struct FrameTab {
    int nframes;
    int after[B2K_MAX_FRAMES]; // ascending; -1 = absolute constant
    int slot[B2K_MAX_FRAMES];
    int kind[B2K_MAX_FRAMES];  // structure class of the tail (b2k_classify34)
    real tail[B2K_MAX_FRAMES][12];
};

template <typename real, int N>
__global__ void __launch_bounds__(128) k_fk_frames(const __grid_constant__ ChainP<real, N> P, const __grid_constant__ FrameTab<real> F,
                                                   const real *__restrict__ q, long long nrows, int ldq,
                                                   real *__restrict__ out, long long row_stride)
{
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= nrows) return;
    const real *qr = q + row * ldq;
    real *orow = out + row * row_stride;
    int f = 0;
    Pose<real> T, U;
    for (; f < F.nframes && F.after[f] < 0; f++) { // constants: the base frame, links that depend on no joint
        pose_from_const(U, F.tail[f]);
        store_pose_row(U, orow + (long long)F.slot[f] * 16);
    }
    pose_from_const(T, P.A[0]); // base folded in by the launcher
#pragma unroll
    for (int j = 0; j < N; j++) {
        if (j > 0) pose_mul_const_right(T, P.A[j], P.akind[j]);
        const real eta = qr[P.jidx[j]] * (P.flip[j] ? (real)-1 : (real)1);
        pose_joint_right(T, P.axis[j], eta, P.trig);
        for (; f < F.nframes && F.after[f] == j; f++) {
            U = T;
            pose_mul_const_right(U, F.tail[f], F.kind[f]);
            store_pose_row(U, orow + (long long)F.slot[f] * 16);
        }
    }
}

template <typename real, int N>
static int frames_launch_n(const b2k_chain_s *c, const real *q, long long nrows, int ldq, const double *base, int nframes,
                           const int32_t *after, const int32_t *slot, const double *tails, real *out, long long nslots,
                           cudaStream_t st)
{
    ChainP<real, N> P;
    b2k_fill_chain<real, N>(c, base, nullptr, true, P);
    for (int f0 = 0; f0 < nframes; f0 += B2K_MAX_FRAMES) {
        FrameTab<real> F;
        F.nframes = nframes - f0 < B2K_MAX_FRAMES ? nframes - f0 : B2K_MAX_FRAMES;
        for (int k = 0; k < F.nframes; k++) {
            double A[12];
            b2k_mat_to34(tails + (size_t)(f0 + k) * 16, A);
            F.after[k] = after[f0 + k];
            F.slot[k] = slot[f0 + k];
            F.kind[k] = b2k_classify34(A);
            for (int e = 0; e < 12; e++) F.tail[k][e] = (real)A[e];
        }
        k_fk_frames<real, N><<<(unsigned)((nrows + 127) / 128), 128, 0, st>>>(P, F, q, nrows, ldq, out, nslots * 16);
        b2k_count_launch();
        B2K_CUDA(cudaGetLastError());
    }
    return B2K_OK;
}

extern "C" int b2k_fkine_frames(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *base, int nframes,
                                const int32_t *after, const int32_t *slot, const double *tails, void *out, int64_t nslots,
                                void *stream)
{
    const char *fn = "b2k_fkine_frames";
    int rc;
    if ((rc = b2k_check_chain(fn, c, dtype, q, N, ldq)) || (rc = b2k_check_affine(fn, "base", base))) return rc;
    if (nframes < 1 || !after || !slot || !tails || nslots < 1) { b2k_set_error("%s: bad frame table", fn); return B2K_ERR_INVALID; }
    for (int k = 0; k < nframes; k++) {
        if (after[k] < -1 || after[k] >= c->n || (k > 0 && after[k] < after[k - 1])) {
            b2k_set_error("%s: after[%d] = %d: must be ascending in [-1, n - 1]", fn, k, after[k]);
            return B2K_ERR_INVALID;
        }
        if (slot[k] < 0 || slot[k] >= nslots) { b2k_set_error("%s: slot[%d] = %d outside [0, %lld)", fn, k, slot[k], (long long)nslots); return B2K_ERR_INVALID; }
        if ((rc = b2k_check_affine(fn, "tail", tails + (size_t)k * 16, k))) return rc;
    }
    if ((rc = b2k_check_array(fn, "out", out, N, 32))) return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(q);
    cudaStream_t st = (cudaStream_t)stream;
    return b2k_for_joints(c->n, [&](auto n) {
        return dtype == B2K_F64 ? frames_launch_n<double, n.value>(c, (const double *)q, N, (int)ldq, base, nframes, after, slot,
                                                                   tails, (double *)out, nslots, st)
                                : frames_launch_n<float, n.value>(c, (const float *)q, N, (int)ldq, base, nframes, after, slot,
                                                                  tails, (float *)out, nslots, st);
    });
}
