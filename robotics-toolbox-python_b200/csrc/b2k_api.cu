// b2k_api.cu -- extern "C" entry points of libb2kin.so (see include/b2kin.h), argument
// validation, error strings, launch accounting and the pipelined host-buffer front ends.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <map>
#include <mutex>
#include <tuple>
#include <vector>

#include "b2k_common.cuh"

// the fkj launchers (b2k_fkj.cuh), one translation unit per dtype
typedef int FkjLaunchFn(const b2k_chain_s *c, int mode, const void *q, long long nrows, long long ldq, const double *base,
                        const double *tool, void *T, void *J, cudaStream_t st);
FkjLaunchFn b2k_fkj_launch_f32, b2k_fkj_launch_f64;

// ------------------------------------------------------------------ error / accounting plumbing
static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void b2k_set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int b2k_check_chain(const char *fn, const b2k_chain_s *c, int dtype, const void *q, int64_t N, int64_t ldq, bool q_on_device)
{
    if (!c) { b2k_set_error("%s: chain handle is NULL", fn); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (c->n < 1 || c->n > B2K_MAX_JOINTS) { b2k_set_error("%s: unsupported joint count %d", fn, c->n); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: N = %lld is negative", fn, (long long)N); return B2K_ERR_INVALID; }
    if (N > 0 && !q) { b2k_set_error("%s: q is NULL", fn); return B2K_ERR_INVALID; }
    if (ldq < c->q_width || ldq > B2K_MAX_QWIDTH) {
        b2k_set_error("%s: q row width %lld outside [%d, %d] (chain reads columns up to %d)", fn, (long long)ldq,
                      c->q_width, B2K_MAX_QWIDTH, c->q_width - 1);
        return B2K_ERR_INVALID;
    }
    return q_on_device ? b2k_check_array(fn, "q", q, N, dtype == B2K_F64 ? 8u : 4u) : B2K_OK;
}

int b2k_check_array(const char *fn, const char *name, const void *p, int64_t N, unsigned align)
{
    if (N > 0 && !p) { b2k_set_error("%s: %s is NULL", fn, name); return B2K_ERR_INVALID; }
    if (((uintptr_t)p) & (align - 1)) { b2k_set_error("%s: %s must be %u-byte aligned", fn, name, align); return B2K_ERR_INVALID; }
    return B2K_OK;
}

int b2k_check_affine(const char *fn, const char *name, const double *M, int index)
{
    if (!M || (M[12] == 0.0 && M[13] == 0.0 && M[14] == 0.0 && M[15] == 1.0)) return B2K_OK;
    if (index < 0) b2k_set_error("%s: %s is not an SE(3)/affine matrix (bottom row must be 0 0 0 1)", fn, name);
    else b2k_set_error("%s: %s %d is not an SE(3)/affine matrix (bottom row must be 0 0 0 1)", fn, name, index);
    return B2K_ERR_INVALID;
}

int b2k_cuda_fail(cudaError_t e, const char *what)
{
    b2k_set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
    return B2K_ERR_CUDA;
}

void b2k_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int b2k_num_sms(int *device_out)
{
    static std::mutex mu;
    static std::map<int, int> cache;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (device_out) *device_out = dev;
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(dev);
    if (it != cache.end()) return it->second;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cache[dev] = sms;
    return sms;
}

int b2k_blocks_per_sm(const void *func, int threads, size_t smem)
{
    static std::mutex mu;
    static std::map<std::tuple<int, const void *, int, size_t>, int> cache;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
    auto key = std::make_tuple(dev, func, threads, smem);
    {
        std::lock_guard<std::mutex> lk(mu);
        auto it = cache.find(key);
        if (it != cache.end()) return it->second;
    }
    cudaError_t e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return b2k_cuda_fail(e, "cudaFuncSetAttribute(MaxDynamicSharedMemorySize)");
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, func, threads, smem);
    if (e != cudaSuccess) return b2k_cuda_fail(e, "cudaOccupancyMaxActiveBlocksPerMultiprocessor");
    std::lock_guard<std::mutex> lk(mu);
    cache[key] = per_sm;
    return per_sm;
}

void b2k_keep_mempool()
{
    static std::mutex mu;
    static std::map<int, bool> done;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return;
    std::lock_guard<std::mutex> lk(mu);
    if (done[dev]) return;
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
        unsigned long long thr = ~0ULL;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    done[dev] = true;
}

extern "C" const char *b2k_last_error(void) { return g_err; }
extern "C" int b2k_version(void) { return B2K_VERSION; }
extern "C" int64_t b2k_launch_count(void) { return (int64_t)g_launches.load(); }

// ------------------------------------------------------------------ forward kinematics and Jacobians
static int fkj_dispatch(const char *fn, b2k_chain_t c, int dtype, int mode, const void *q, int64_t N, int64_t ldq,
                        const double *base, const double *tool, void *T, void *J, void *stream)
{
    int rc;
    if ((rc = b2k_check_chain(fn, c, dtype, q, N, ldq)) || (rc = b2k_check_affine(fn, "base", base)) ||
        (rc = b2k_check_affine(fn, "tool", tool)))
        return rc;
    // T is stored in 32-byte pieces; J leaves through a shared-memory stage of 6n-element rows (TileStage in b2k_fkj.cuh)
    const int es = dtype == B2K_F64 ? 8 : 4;
    if ((mode & FKJ_T) && (rc = b2k_check_array(fn, "T", T, N, 32))) return rc;
    if ((mode & (FKJ_J0 | FKJ_JE)) && (rc = b2k_check_array(fn, "J", J, N, b2k_stage_unit(6 * c->n * es)))) return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(q);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == B2K_F64) return b2k_fkj_launch_f64(c, mode, q, N, ldq, base, tool, T, J, st);
    return b2k_fkj_launch_f32(c, mode, q, N, ldq, base, tool, T, J, st);
}

extern "C" int b2k_fkine(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *base,
                         const double *tool, void *T, void *stream)
{
    return fkj_dispatch("b2k_fkine", c, dtype, FKJ_T, q, N, ldq, base, tool, T, nullptr, stream);
}

extern "C" int b2k_jacob0(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *tool, void *J,
                          void *stream)
{
    return fkj_dispatch("b2k_jacob0", c, dtype, FKJ_J0, q, N, ldq, nullptr, tool, nullptr, J, stream);
}

extern "C" int b2k_jacobe(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *tool, void *J,
                          void *stream)
{
    return fkj_dispatch("b2k_jacobe", c, dtype, FKJ_JE, q, N, ldq, nullptr, tool, nullptr, J, stream);
}

extern "C" int b2k_fkine_jacob0(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *base,
                                const double *tool, void *T, void *J, void *stream)
{
    return fkj_dispatch("b2k_fkine_jacob0", c, dtype, FKJ_T | FKJ_J0, q, N, ldq, base, tool, T, J, stream);
}

extern "C" int b2k_fkine_jacobe(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *base,
                                const double *tool, void *T, void *J, void *stream)
{
    return fkj_dispatch("b2k_fkine_jacobe", c, dtype, FKJ_T | FKJ_JE, q, N, ldq, base, tool, T, J, stream);
}

// ------------------------------------------------------------------ operations on an rne handle
// the generic kernels (b2k_rne.cuh), one translation unit per family of operations and dtype
typedef int RneGenericFn(const b2k_rne_s *, int op, int dtype, const b2k_rne_args &, cudaStream_t);
RneGenericFn b2k_rne_generic_rne, b2k_rne_generic_wrench, b2k_rne_generic_fan_f32, b2k_rne_generic_fan_f64,
    b2k_rne_generic_deriv_f32, b2k_rne_generic_deriv_f64, b2k_rne_generic_regressor_f32, b2k_rne_generic_regressor_f64;

// Every argument is checked against the operation's row of B2K_RNE_OPS before any CUDA call; then the robot-specialised
// kernel (b2k_rne_spec.cu) serves the full 32-row tiles of the operations it has, and the generic kernel the rest.
// The checks of an operation's handle, scalars and inputs (its row of B2K_RNE_OPS), in this order
static int rne_check_inputs(const char *fn, int op, b2k_rne_t r, int dtype, const b2k_rne_args &a)
{
    const b2k_rne_op_s &d = B2K_RNE_OPS[op];
    if (!r) { b2k_set_error("%s: rne handle is NULL", fn); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (a.nrows < 0) { b2k_set_error("%s: N is negative", fn); return B2K_ERR_INVALID; }
    if (r->n < 1 || r->n > B2K_MAX_JOINTS) { b2k_set_error("%s: unsupported joint count %d", fn, r->n); return B2K_ERR_INVALID; }
    if (d.grav && !a.grav) { b2k_set_error("%s: grav is NULL (pass -robot.gravity like DHRobot.rne)", fn); return B2K_ERR_INVALID; }
    int rc;
    const int es = dtype == B2K_F64 ? 8 : 4;
    for (int i = 0; i < d.nin; i++)
        if ((rc = b2k_check_array(fn, d.in[i], a.in[i], a.nrows, es))) return rc;
    return B2K_OK;
}

static int rne_dispatch(const char *fn, int op, b2k_rne_t r, int dtype, b2k_rne_args a, void *stream)
{
    const b2k_rne_op_s &d = B2K_RNE_OPS[op];
    int rc;
    if ((rc = rne_check_inputs(fn, op, r, dtype, a))) return rc;
    const int es = dtype == B2K_F64 ? 8 : 4;
    // each output leaves through a per-warp stage of its rows, copied in b2k_stage_unit(row bytes) pieces (b2k_rne.cuh)
    for (int o = 0; o < d.nout; o++)
        if ((rc = b2k_check_array(fn, d.out[o], a.out[o], a.nrows, b2k_stage_unit(d.out_row(o, r->n) * es)))) return rc;
    if (a.nrows == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(a.in[0]);
    cudaStream_t st = (cudaStream_t)stream;
    if (op <= B2K_GEN_RNE_WRENCH) {
        const long long done = b2k_rne_spec_launch(r, op, dtype, a.in[0], a.in[1], a.in[2], a.nrows, a.grav, a.fext, a.out[0], a.out[1], st);
        if (done < 0) return (int)done;
        if (done == a.nrows) return B2K_OK;
        for (int i = 0; i < d.nin; i++) a.in[i] = (const char *)a.in[i] + (size_t)done * r->n * es;
        for (int o = 0; o < d.nout; o++) a.out[o] = (char *)a.out[o] + (size_t)done * d.out_row(o, r->n) * es;
        a.nrows -= done;
    }
    const bool f64 = dtype == B2K_F64;
    RneGenericFn *generic = op == B2K_GEN_RNE             ? b2k_rne_generic_rne
                            : op == B2K_GEN_RNE_WRENCH    ? b2k_rne_generic_wrench
                            : op == B2K_GEN_RNE_REGRESSOR ? (f64 ? b2k_rne_generic_regressor_f64 : b2k_rne_generic_regressor_f32)
                            : op >= B2K_GEN_RNE_DERIV     ? (f64 ? b2k_rne_generic_deriv_f64 : b2k_rne_generic_deriv_f32)
                                                          : (f64 ? b2k_rne_generic_fan_f64 : b2k_rne_generic_fan_f32);
    return generic(r, op, dtype, a, st);
}

extern "C" int b2k_rne(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                       const double *grav, const double *fext, void *tau, void *stream)
{
    return rne_dispatch("b2k_rne", B2K_GEN_RNE, r, dtype, {{q, qd, qdd}, {tau}, N, grav, fext}, stream);
}

extern "C" int b2k_rne_wrench(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                              const double *grav, const double *fext, void *tau, void *wbase, void *stream)
{
    return rne_dispatch("b2k_rne_wrench", B2K_GEN_RNE_WRENCH, r, dtype, {{q, qd, qdd}, {tau, wbase}, N, grav, fext}, stream);
}

// ------------------------------------------------------------------ host-buffer front ends
extern "C" int b2k_host_alloc(void **ptr, int64_t bytes)
{
    if (!ptr || bytes < 0) { b2k_set_error("b2k_host_alloc: bad arguments"); return B2K_ERR_INVALID; }
    *ptr = nullptr;
    if (bytes == 0) return B2K_OK;
    B2K_CUDA(cudaHostAlloc(ptr, (size_t)bytes, cudaHostAllocPortable));
    return B2K_OK;
}

extern "C" int b2k_host_free(void *ptr)
{
    if (ptr) B2K_CUDA(cudaFreeHost(ptr));
    return B2K_OK;
}

namespace {
// A small pool of per-device pipeline slots (device staging buffers + stream), reused across calls.
struct Slot {
    cudaStream_t st = nullptr;
    cudaEvent_t h2d_done = nullptr; // recorded behind the slot's H2D copies: its bounce buffers are free again after it
    void *d_in[3] = {nullptr, nullptr, nullptr};
    void *d_out[2] = {nullptr, nullptr};
    void *h_stage[3] = {nullptr, nullptr, nullptr}; // pinned bounce buffers for PAGEABLE caller inputs
    size_t in_cap[3] = {0, 0, 0}, out_cap[2] = {0, 0}, stage_cap[3] = {0, 0, 0};
    bool h2d_pending = false;
};
struct Pipe {
    std::mutex mu; // one pass at a time per device; passes on different devices run concurrently
    std::vector<Slot> slots;
};
std::mutex g_pipe_mu; // guards the map only
std::map<int, Pipe> g_pipes;

int ensure(void **p, size_t *cap, size_t need)
{
    if (*cap >= need) return B2K_OK;
    if (*p) cudaFree(*p);
    *p = nullptr;
    *cap = 0;
    B2K_CUDA(cudaMalloc(p, need));
    *cap = need;
    return B2K_OK;
}

int ensure_host(void **p, size_t *cap, size_t need)
{
    if (*cap >= need) return B2K_OK;
    if (*p) cudaFreeHost(*p);
    *p = nullptr;
    *cap = 0;
    B2K_CUDA(cudaHostAlloc(p, need, cudaHostAllocPortable));
    *cap = need;
    return B2K_OK;
}

// true when the driver cannot DMA from this host pointer directly (ordinary malloc / numpy memory)
bool is_pageable(const void *p)
{
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
}

constexpr int kSlots = 3;
constexpr long long kChunkRows = 1 << 17; // 128k rows per chunk: ~60 MB of Panda fp64 output

// Generic chunked pipeline: for each chunk, H2D the inputs, run `kernel`, D2H the outputs, round-robin
// over kSlots streams so the copy engines and the SMs overlap.  Inputs in pageable memory (what a numpy
// caller of the reference API holds) are staged by this thread into a pinned bounce buffer of the slot
// and copied from there: a cudaMemcpyAsync straight from pageable memory would block the host until the
// driver has staged it, serialising the pipeline; the explicit stage costs one memcpy that hides behind
// the D2H traffic of the previous chunks.
template <typename F>
int run_pipeline(int device, long long N, int n_in, const void *const *h_in, const size_t *in_row_bytes, int n_out,
                 void *const *h_out, const size_t *out_row_bytes, F kernel)
{
    DeviceGuard guard(device, true); // restores the caller's device on every exit path
    if (guard.rc) return guard.rc;
    Pipe *pp;
    {
        std::lock_guard<std::mutex> lk(g_pipe_mu);
        pp = &g_pipes[device]; // std::map nodes are stable
    }
    Pipe &P = *pp;
    std::lock_guard<std::mutex> lk(P.mu);
    if (P.slots.empty()) { // create every stream / event first; publish the slots only when all of them exist
        std::vector<Slot> fresh(kSlots);
        cudaError_t e = cudaSuccess;
        for (auto &s : fresh) {
            e = cudaStreamCreateWithFlags(&s.st, cudaStreamNonBlocking);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.h2d_done, cudaEventDisableTiming);
            if (e != cudaSuccess) break;
        }
        if (e != cudaSuccess) {
            for (auto &t : fresh) {
                if (t.h2d_done) cudaEventDestroy(t.h2d_done);
                if (t.st) cudaStreamDestroy(t.st);
            }
            return b2k_cuda_fail(e, "creating the pipeline streams");
        }
        P.slots = std::move(fresh);
    }
    bool pageable[3] = {false, false, false};
    for (int i = 0; i < n_in; i++) pageable[i] = is_pageable(h_in[i]);
    const long long chunk = N < kChunkRows ? N : kChunkRows;
    int rc = B2K_OK;
    long long done = 0;
    int k = 0;
    while (done < N && rc == B2K_OK) {
        Slot &s = P.slots[k % kSlots];
        const long long rows = (N - done) < chunk ? (N - done) : chunk;
        bool staged = false;
        for (int i = 0; i < n_in && rc == B2K_OK; i++) {
            rc = ensure(&s.d_in[i], &s.in_cap[i], (size_t)chunk * in_row_bytes[i]);
            if (rc) break;
            const char *src = (const char *)h_in[i] + (size_t)done * in_row_bytes[i];
            const size_t bytes = (size_t)rows * in_row_bytes[i];
            if (pageable[i]) {
                if ((rc = ensure_host(&s.h_stage[i], &s.stage_cap[i], (size_t)chunk * in_row_bytes[i]))) break;
                if (s.h2d_pending) { // the previous chunk of this slot may still be reading the bounce buffers
                    cudaError_t e = cudaEventSynchronize(s.h2d_done);
                    if (e != cudaSuccess) { rc = b2k_cuda_fail(e, "cudaEventSynchronize"); break; }
                    s.h2d_pending = false;
                }
                memcpy(s.h_stage[i], src, bytes);
                src = (const char *)s.h_stage[i];
                staged = true;
            }
            cudaError_t e = cudaMemcpyAsync(s.d_in[i], src, bytes, cudaMemcpyHostToDevice, s.st);
            if (e != cudaSuccess) rc = b2k_cuda_fail(e, "cudaMemcpyAsync H2D");
        }
        if (staged && rc == B2K_OK) {
            cudaError_t e = cudaEventRecord(s.h2d_done, s.st);
            if (e != cudaSuccess) rc = b2k_cuda_fail(e, "cudaEventRecord");
            s.h2d_pending = true;
        }
        for (int i = 0; i < n_out && rc == B2K_OK; i++) rc = ensure(&s.d_out[i], &s.out_cap[i], (size_t)chunk * out_row_bytes[i]);
        if (rc == B2K_OK) rc = kernel(s, rows);
        for (int i = 0; i < n_out && rc == B2K_OK; i++) {
            cudaError_t e = cudaMemcpyAsync((char *)h_out[i] + (size_t)done * out_row_bytes[i], s.d_out[i],
                                            (size_t)rows * out_row_bytes[i], cudaMemcpyDeviceToHost, s.st);
            if (e != cudaSuccess) rc = b2k_cuda_fail(e, "cudaMemcpyAsync D2H");
        }
        done += rows;
        k++;
    }
    for (auto &s : P.slots) {
        cudaError_t e = cudaStreamSynchronize(s.st);
        if (e != cudaSuccess && rc == B2K_OK) rc = b2k_cuda_fail(e, "cudaStreamSynchronize");
        s.h2d_pending = false;
    }
    return rc;
}
} // namespace

// b2k_fkine_host and b2k_fkine_jacob0_host (jacob: also J (N, 6, n))
static int fkine_host(const char *fn, b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *base,
                      const double *tool, void *T, bool jacob, void *J, int device)
{
    int rc;
    if ((rc = b2k_check_chain(fn, c, dtype, q, N, ldq, false)) || (rc = b2k_check_array(fn, "T", T, N, 1)) ||
        (jacob && (rc = b2k_check_array(fn, "J", J, N, 1))))
        return rc;
    if (N == 0) return B2K_OK;
    const size_t es = dtype == B2K_F64 ? 8 : 4;
    const void *h_in[1] = {q};
    size_t in_b[1] = {(size_t)ldq * es};
    void *h_out[2] = {T, J};
    size_t out_b[2] = {16 * es, (size_t)6 * c->n * es};
    return run_pipeline(device, N, 1, h_in, in_b, jacob ? 2 : 1, h_out, out_b, [&](Slot &s, long long rows) {
        if (jacob) return b2k_fkine_jacob0(c, dtype, s.d_in[0], rows, ldq, base, tool, s.d_out[0], s.d_out[1], s.st);
        return b2k_fkine(c, dtype, s.d_in[0], rows, ldq, base, tool, s.d_out[0], s.st);
    });
}

extern "C" int b2k_fkine_jacob0_host(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *base,
                                     const double *tool, void *T, void *J, int device)
{
    return fkine_host("b2k_fkine_jacob0_host", c, dtype, q, N, ldq, base, tool, T, true, J, device);
}

extern "C" int b2k_fkine_host(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *base,
                              const double *tool, void *T, int device)
{
    return fkine_host("b2k_fkine_host", c, dtype, q, N, ldq, base, tool, T, false, nullptr, device);
}

// b2k_rne_host and b2k_rne_wrench_host (wrench: also the base wrench wbase (N, 6))
static int rne_host(const char *fn, b2k_rne_t r, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                    const double *grav, const double *fext, void *tau, bool wrench, void *wbase, int device)
{
    if (!r) { b2k_set_error("%s: rne handle is NULL", fn); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (N < 0 || (N > 0 && (!q || !qd || !qdd || !tau || !grav))) { b2k_set_error("%s: NULL argument", fn); return B2K_ERR_INVALID; }
    const size_t es = dtype == B2K_F64 ? 8 : 4;
    int rc;
    if (wrench && (rc = b2k_check_array(fn, "wbase", wbase, N, (unsigned)es))) return rc;
    if (N == 0) return B2K_OK;
    const void *h_in[3] = {q, qd, qdd};
    size_t in_b[3] = {r->n * es, r->n * es, r->n * es};
    void *h_out[2] = {tau, wbase};
    size_t out_b[2] = {r->n * es, 6 * es};
    return run_pipeline(device, N, 3, h_in, in_b, wrench ? 2 : 1, h_out, out_b, [&](Slot &s, long long rows) {
        if (wrench) return b2k_rne_wrench(r, dtype, s.d_in[0], s.d_in[1], s.d_in[2], rows, grav, fext, s.d_out[0], s.d_out[1], s.st);
        return b2k_rne(r, dtype, s.d_in[0], s.d_in[1], s.d_in[2], rows, grav, fext, s.d_out[0], s.st);
    });
}

extern "C" int b2k_rne_host(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                            const double *grav, const double *fext, void *tau, int device)
{
    return rne_host("b2k_rne_host", r, dtype, q, qd, qdd, N, grav, fext, tau, false, nullptr, device);
}

extern "C" int b2k_rne_wrench_host(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                                   const double *grav, const double *fext, void *tau, void *wbase, int device)
{
    return rne_host("b2k_rne_wrench_host", r, dtype, q, qd, qdd, N, grav, fext, tau, true, wbase, device);
}

// ------------------------------------------------------------------ inverse kinematics
// the launchers (b2k_ik.cuh), one translation unit per family of kernels and dtype
typedef int IkLaunchFn(const b2k_chain_s *, const IkArgs &, cudaStream_t);
IkLaunchFn b2k_ik_launch_f32, b2k_ik_launch_f64, b2k_ik_nr_launch_f32, b2k_ik_nr_launch_f64, b2k_ik_ns_launch_f32,
    b2k_ik_ns_launch_f64, b2k_ik_qp_launch_f32, b2k_ik_qp_launch_f64;

enum { IK_LM, IK_NULL, IK_QP }; // b2k_ik_lm, b2k_ikine_null, b2k_ikine_qp

// Every argument of the three IK entry points is checked before any CUDA call; then the variant and the method pick the
// translation unit.
static int ik_dispatch(const char *fn, int variant, b2k_chain_t c, int dtype, IkArgs a, void *stream)
{
    if (!c) { b2k_set_error("%s: chain handle is NULL", fn); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (a.N < 0) { b2k_set_error("%s: N is negative", fn); return B2K_ERR_INVALID; }
    // The solver works on the chain's own joint vector (q0 and q_out hold the n joints in chain order, i.e.
    // q[ets.jindices] -- what IKSolver.solve hands back, IK.py:216-240,346); a sub-chain of a larger robot
    // (jindices 3..6, say) is therefore served as it is.  Two joints driven by one coordinate are not.
    if (!c->distinct_jindex) {
        b2k_set_error("%s: two joints of the chain share a jindex (coupled joints are outside the solver's model)", fn);
        return B2K_ERR_INVALID;
    }
    if (variant == IK_NULL && (c->n < 7 || c->n > B2K_MAX_JOINTS)) {
        b2k_set_error("%s: the null-space terms need a redundant chain of 7..%d joints (n = %d)", fn, B2K_MAX_JOINTS, c->n);
        return B2K_ERR_INVALID;
    }
    if (variant == IK_QP && (c->n < 1 || c->n > B2K_MAX_JOINTS)) { b2k_set_error("%s: unsupported joint count %d", fn, c->n); return B2K_ERR_INVALID; }
    if (a.ilimit < 1 || a.slimit < 1) { b2k_set_error("%s: ilimit and slimit must be >= 1", fn); return B2K_ERR_INVALID; }
    if (variant != IK_QP && (a.method < B2K_LM_CHAN || a.method > B2K_IK_GN)) { b2k_set_error("%s: bad method %d", fn, a.method); return B2K_ERR_INVALID; }
    if (variant == IK_LM && a.semantics != B2K_IK_SEM_CPP && a.semantics != B2K_IK_SEM_PYTHON) {
        b2k_set_error("%s: bad semantics %d", fn, a.semantics);
        return B2K_ERR_INVALID;
    }
    const auto &g = a.gains;
    if (variant == IK_NULL) {
        if (!isfinite(g.kq) || !isfinite(g.km)) { b2k_set_error("%s: kq and km must be finite", fn); return B2K_ERR_INVALID; }
        if (!(g.kq > 0) && !(g.km > 0)) { b2k_set_error("%s: at least one of kq and km must be > 0", fn); return B2K_ERR_INVALID; }
        if (!isfinite(g.ps)) { b2k_set_error("%s: ps must be finite", fn); return B2K_ERR_INVALID; }
    }
    if (variant == IK_QP) {
        if (!isfinite(g.kj) || !isfinite(g.ks) || !isfinite(g.kq) || !isfinite(g.km) || !isfinite(g.ps)) {
            b2k_set_error("%s: kj, ks, kq, km and ps must be finite", fn);
            return B2K_ERR_INVALID;
        }
        if (!(g.kj > 0) || !(g.ks > 0)) {
            b2k_set_error("%s: kj and ks must be > 0 (the step's quadratic form is not positive definite otherwise)", fn);
            return B2K_ERR_INVALID;
        }
    }
    // pi: read by the null-space terms always, by the QP step only for its velocity damper (kq > 0)
    if (variant == IK_NULL || (variant == IK_QP && g.kq > 0)) {
        if (!g.pi) { b2k_set_error("%s: pi is NULL", fn); return B2K_ERR_INVALID; }
        for (int i = 0; i < c->n; i++) {
            if (!isfinite(g.pi[i])) { b2k_set_error("%s: pi[%d] is not finite", fn, i); return B2K_ERR_INVALID; }
            if (g.kq > 0 && g.ps == g.pi[i]) {
                b2k_set_error("%s: ps == pi[%d] divides by zero in the %s", fn, i,
                              variant == IK_NULL ? "joint-limit term" : "velocity damper");
                return B2K_ERR_INVALID;
            }
        }
    }
    if (variant == IK_QP && g.km > 0 && c->n < 6) {
        b2k_set_error("%s: km > 0 needs at least 6 joints (n = %d): J J^T is singular for fewer", fn, c->n);
        return B2K_ERR_INVALID;
    }
    int rc;
    if ((rc = b2k_check_array(fn, "Tep", a.Tep, a.N, 8)) || (rc = b2k_check_array(fn, "q_out", a.q_out, a.N, 8)) ||
        (rc = b2k_check_array(fn, "success", a.success, a.N, 8)) ||
        (rc = b2k_check_array(fn, "iterations", a.iterations, a.N, 8)) ||
        (rc = b2k_check_array(fn, "searches", a.searches, a.N, 8)) ||
        (rc = b2k_check_array(fn, "residual", a.residual, a.N, 8)))
        return rc;
    const bool pinv = variant != IK_QP && (a.method == B2K_IK_NR || a.method == B2K_IK_GN);
    if (pinv && a.lambda < 0) { b2k_set_error("%s: pinv_damping is negative", fn); return B2K_ERR_INVALID; }
    if (a.N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(a.Tep);
    // What the kernels read of lambda, method and semantics: GN takes the undamped pseudo-inverse step, the QP step is
    // neither damped nor weighted, and the null-space terms and the QP step run in the Python solver loop only.
    if (variant == IK_QP) a.lambda = 0.0, a.method = 0;
    else if (a.method == B2K_IK_GN) a.lambda = 0.0;
    if (variant != IK_LM) a.semantics = B2K_IK_SEM_PYTHON;
    const bool f64 = dtype == B2K_F64;
    IkLaunchFn *launch = variant == IK_QP     ? (f64 ? b2k_ik_qp_launch_f64 : b2k_ik_qp_launch_f32)
                         : variant == IK_NULL ? (f64 ? b2k_ik_ns_launch_f64 : b2k_ik_ns_launch_f32)
                         : pinv               ? (f64 ? b2k_ik_nr_launch_f64 : b2k_ik_nr_launch_f32)
                                              : (f64 ? b2k_ik_launch_f64 : b2k_ik_launch_f32);
    return launch(c, a, (cudaStream_t)stream);
}

extern "C" int b2k_ik_lm(b2k_chain_t c, int dtype, const void *Tep, int64_t N, const void *q0, int ilimit, int slimit,
                         double tol, int reject_jl, const double *we, double lambda, int method, uint64_t seed,
                         int semantics, int rng_per_row, void *q_out, int32_t *success, int32_t *iterations,
                         int32_t *searches, void *residual, void *stream)
{
    return ik_dispatch("b2k_ik_lm", IK_LM, c, dtype,
                       {Tep, q0, q_out, success, iterations, searches, residual, N, ilimit, slimit, tol, reject_jl, we,
                        lambda, method, seed, semantics, rng_per_row, {}},
                       stream);
}

extern "C" int b2k_ikine_null(b2k_chain_t c, int dtype, const void *Tep, int64_t N, const void *q0, int ilimit,
                              int slimit, double tol, int reject_jl, const double *we, double lambda, int method,
                              uint64_t seed, int rng_per_row, double kq, double km, double ps, const double *pi,
                              void *q_out, int32_t *success, int32_t *iterations, int32_t *searches, void *residual,
                              void *stream)
{
    return ik_dispatch("b2k_ikine_null", IK_NULL, c, dtype,
                       {Tep, q0, q_out, success, iterations, searches, residual, N, ilimit, slimit, tol, reject_jl, we,
                        lambda, method, seed, 0, rng_per_row, {0.0, 0.0, kq, km, ps, pi}},
                       stream);
}

extern "C" int b2k_ikine_qp(b2k_chain_t c, int dtype, const void *Tep, int64_t N, const void *q0, int ilimit,
                            int slimit, double tol, int reject_jl, const double *we, uint64_t seed, int rng_per_row,
                            double kj, double ks, double kq, double km, double ps, const double *pi, void *q_out,
                            int32_t *success, int32_t *iterations, int32_t *searches, void *residual, void *stream)
{
    return ik_dispatch("b2k_ikine_qp", IK_QP, c, dtype,
                       {Tep, q0, q_out, success, iterations, searches, residual, N, ilimit, slimit, tol, reject_jl, we,
                        0.0, 0, seed, 0, rng_per_row, {kj, ks, kq, km, ps, pi}},
                       stream);
}

// ------------------------------------------------------------------ dynamics fan-outs
extern "C" int b2k_rne_inertia(b2k_rne_t r, int dtype, const void *q, int64_t N, void *M, void *stream)
{
    return rne_dispatch("b2k_rne_inertia", B2K_GEN_INERTIA, r, dtype, {{q}, {M}, N, nullptr, nullptr}, stream);
}
extern "C" int b2k_rne_gravload(b2k_rne_t r, int dtype, const void *q, int64_t N, const double *grav, void *taug, void *stream)
{
    return rne_dispatch("b2k_rne_gravload", B2K_GEN_GRAVLOAD, r, dtype, {{q}, {taug}, N, grav, nullptr}, stream);
}
extern "C" int b2k_rne_itorque(b2k_rne_t r, int dtype, const void *q, const void *qdd, int64_t N, void *taui, void *stream)
{
    return rne_dispatch("b2k_rne_itorque", B2K_GEN_ITORQUE, r, dtype, {{q, qdd}, {taui}, N, nullptr, nullptr}, stream);
}
extern "C" int b2k_rne_coriolis(b2k_rne_t r, int dtype, const void *q, const void *qd, int64_t N, void *Cm, void *stream)
{
    return rne_dispatch("b2k_rne_coriolis", B2K_GEN_CORIOLIS, r, dtype, {{q, qd}, {Cm}, N, nullptr, nullptr}, stream);
}
extern "C" int b2k_rne_accel(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *torque, int64_t N,
                             const double *grav, void *qdd, void *stream)
{
    return rne_dispatch("b2k_rne_accel", B2K_GEN_ACCEL, r, dtype, {{q, qd, torque}, {qdd}, N, grav, nullptr}, stream);
}

// ------------------------------------------------------------------ analytical derivatives of the recursion (b2k_rne.cuh)
extern "C" int b2k_rne_derivatives(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                                   const double *grav, const double *fext, void *dtau_dq, void *dtau_dqd, void *stream)
{
    return rne_dispatch("b2k_rne_derivatives", B2K_GEN_RNE_DERIV, r, dtype, {{q, qd, qdd}, {dtau_dq, dtau_dqd}, N, grav, fext},
                        stream);
}

extern "C" int b2k_rne_accel_derivatives(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *torque, int64_t N,
                                         const double *grav, void *dqdd_dq, void *dqdd_dqd, void *dqdd_dtau, void *stream)
{
    return rne_dispatch("b2k_rne_accel_derivatives", B2K_GEN_ACCEL_DERIV, r, dtype,
                        {{q, qd, torque}, {dqdd_dq, dqdd_dqd, dqdd_dtau}, N, grav, nullptr}, stream);
}

// ------------------------------------------------------------------ the dynamics regressor and its normal equations (b2k_rne.cuh)
extern "C" int b2k_rne_regressor(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                                 const double *grav, void *Y, void *stream)
{
    return rne_dispatch("b2k_rne_regressor", B2K_GEN_RNE_REGRESSOR, r, dtype, {{q, qd, qdd}, {Y}, N, grav, nullptr}, stream);
}

int b2k_rne_regressor_gram_f32(const b2k_rne_s *, const b2k_rne_args &, const void *, const double *, double *, double *,
                               double *, cudaStream_t);
int b2k_rne_regressor_gram_f64(const b2k_rne_s *, const b2k_rne_args &, const void *, const double *, double *, double *,
                               double *, cudaStream_t);

extern "C" int b2k_rne_regressor_gram(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *qdd, const void *tau,
                                      int64_t N, const double *grav, const double *weights, double *G, double *b, double *s,
                                      void *stream)
{
    const char *fn = "b2k_rne_regressor_gram";
    const b2k_rne_args a = {{q, qd, qdd}, {nullptr}, N, grav, nullptr};
    int rc;
    if ((rc = rne_check_inputs(fn, B2K_GEN_RNE_REGRESSOR, r, dtype, a))) return rc;
    if ((rc = b2k_check_array(fn, "tau", tau, N, dtype == B2K_F64 ? 8 : 4))) return rc;
    if (weights)
        for (int j = 0; j < r->n; j++)
            if (!isfinite(weights[j]) || weights[j] < 0) {
                b2k_set_error("%s: weights[%d] = %g is not a finite value >= 0", fn, j, weights[j]);
                return B2K_ERR_INVALID;
            }
    // the sums are written whatever N is (zeros for N = 0)
    if ((rc = b2k_check_array(fn, "G", G, 1, 8)) || (rc = b2k_check_array(fn, "b", b, 1, 8)) || (rc = b2k_check_array(fn, "s", s, 1, 8)))
        return rc;
    B2K_ON_DEVICE_OF(G);
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) {
        const size_t p = 14 * (size_t)r->n;
        B2K_CUDA(cudaMemsetAsync(G, 0, p * p * sizeof(double), st));
        B2K_CUDA(cudaMemsetAsync(b, 0, p * sizeof(double), st));
        B2K_CUDA(cudaMemsetAsync(s, 0, sizeof(double), st));
        return B2K_OK;
    }
    return dtype == B2K_F64 ? b2k_rne_regressor_gram_f64(r, a, tau, weights, G, b, s, st)
                            : b2k_rne_regressor_gram_f32(r, a, tau, weights, G, b, s, st);
}
