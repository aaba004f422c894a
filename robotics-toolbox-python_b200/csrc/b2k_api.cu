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

// per-dtype launchers (b2k_fkj_f32.cu / b2k_fkj_f64.cu / b2k_rne.cu / b2k_ik_*.cu)
int b2k_fkj_launch_f32(const b2k_chain_s *, int, const void *, long long, long long, const double *, const double *,
                       void *, void *, cudaStream_t);
int b2k_fkj_launch_f64(const b2k_chain_s *, int, const void *, long long, long long, const double *, const double *,
                       void *, void *, cudaStream_t);
int b2k_fkw_launch(const b2k_chain_s *, int dtype, int mode, const void *, long long, long long, const double *,
                   const double *, void *, void *, cudaStream_t);
int b2k_rne_launch(const b2k_rne_s *, int dtype, const void *, const void *, const void *, long long, const double *,
                   const double *, void *, cudaStream_t);
int b2k_rne_wrench_launch(const b2k_rne_s *, int dtype, const void *, const void *, const void *, long long, const double *,
                          const double *, void *, void *, cudaStream_t);

enum { FKJ_T = 1, FKJ_J0 = 2, FKJ_JE = 4 };

// ------------------------------------------------------------------ error / accounting plumbing
static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};
static std::atomic<int> g_variant{0};

void b2k_set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int b2k_cuda_fail(cudaError_t e, const char *what)
{
    b2k_set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
    return B2K_ERR_CUDA;
}

void b2k_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int b2k_get_variant() { return g_variant.load(std::memory_order_relaxed); }

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

int b2k_tiles_per_warp(bool with_jacobian)
{
    static const int pose = [] { const char *e = getenv("B2K_TPW_POSE"); int v = e ? atoi(e) : 1; return v < 1 ? 1 : v; }();
    static const int jac = [] { const char *e = getenv("B2K_TPW_JAC"); int v = e ? atoi(e) : 1; return v < 1 ? 1 : v; }();
    return with_jacobian ? jac : pose;
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
extern "C" int b2k_set_variant(int v)
{
    if (v < 0 || v > 4) { b2k_set_error("b2k_set_variant: variant must be 0..4"); return B2K_ERR_INVALID; }
    g_variant.store(v);
    return B2K_OK;
}

// ------------------------------------------------------------------ validation helpers
// q_on_device: the pointer is read by a kernel (element-wise at worst: only the natural alignment of the element
// type is needed); host pointers of the *_host front ends only go through cudaMemcpy and need none.
static int check_common(const char *fn, const b2k_chain_s *c, int dtype, const void *q, int64_t N, int64_t ldq,
                        bool q_on_device = true)
{
    if (!c) { b2k_set_error("%s: chain handle is NULL", fn); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: N = %lld is negative", fn, (long long)N); return B2K_ERR_INVALID; }
    if (N > 0 && !q) { b2k_set_error("%s: q is NULL", fn); return B2K_ERR_INVALID; }
    if (ldq < c->q_width || ldq > B2K_MAX_QWIDTH) {
        b2k_set_error("%s: q row width %lld outside [%d, %d] (chain reads columns up to %d)", fn, (long long)ldq,
                      c->q_width, B2K_MAX_QWIDTH, c->q_width - 1);
        return B2K_ERR_INVALID;
    }
    const unsigned es = dtype == B2K_F64 ? 8u : 4u;
    if (q_on_device && (((uintptr_t)q) & (es - 1))) { b2k_set_error("%s: q must be %u-byte aligned", fn, es); return B2K_ERR_INVALID; }
    return B2K_OK;
}

static int check_out(const char *fn, const char *name, const void *p, int64_t N, unsigned align = 8)
{
    if (N > 0 && !p) { b2k_set_error("%s: %s is NULL", fn, name); return B2K_ERR_INVALID; }
    if (align > 1 && (((uintptr_t)p) & (align - 1))) { b2k_set_error("%s: %s must be %u-byte aligned", fn, name, align); return B2K_ERR_INVALID; }
    return B2K_OK;
}

static int check_affine(const char *fn, const char *name, const double *M)
{
    if (M && (M[12] != 0.0 || M[13] != 0.0 || M[14] != 0.0 || M[15] != 1.0)) {
        b2k_set_error("%s: %s is not an SE(3)/affine matrix (bottom row must be 0 0 0 1)", fn, name);
        return B2K_ERR_INVALID;
    }
    return B2K_OK;
}

static int fkj_dispatch(const char *fn, b2k_chain_t c, int dtype, int mode, const void *q, int64_t N, int64_t ldq,
                        const double *base, const double *tool, void *T, void *J, void *stream)
{
    int rc = check_common(fn, c, dtype, q, N, ldq);
    if (rc) return rc;
    // T is stored in 32-byte pieces; J leaves through a shared-memory stage whose copy unit (TileStage<real, 6n>::UB in
    // b2k_fkj.cuh) is 16 bytes when a 6n-element row is a whole number of 16-byte units, else 8
    const unsigned es = dtype == B2K_F64 ? 8u : 4u;
    const unsigned jub = (6u * (unsigned)c->n * es) % 16u == 0 ? 16u : 8u;
    if ((mode & FKJ_T) && (rc = check_out(fn, "T", T, N, 32))) return rc;
    if ((mode & (FKJ_J0 | FKJ_JE)) && (rc = check_out(fn, "J", J, N, jub))) return rc;
    if ((rc = check_affine(fn, "base", base)) || (rc = check_affine(fn, "tool", tool))) return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(q);
    cudaStream_t st = (cudaStream_t)stream;
    if (b2k_get_variant() == 1 && !(mode & FKJ_JE))
        return b2k_fkw_launch(c, dtype, mode, q, N, ldq, base, tool, T, J, st);
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

// b2k_rne and b2k_rne_wrench (wrench: also the base wrench, wbase (N, 6)); every argument is checked before any CUDA call
static int rne_run(const char *fn, b2k_rne_t r, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                   const double *grav, const double *fext, void *tau, bool wrench, void *wbase, void *stream)
{
    if (!r) { b2k_set_error("%s: rne handle is NULL", fn); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: N is negative", fn); return B2K_ERR_INVALID; }
    if (!grav) { b2k_set_error("%s: grav is NULL (pass -robot.gravity like DHRobot.rne)", fn); return B2K_ERR_INVALID; }
    int rc;
    const unsigned es = dtype == B2K_F64 ? 8u : 4u;
    if ((rc = check_out(fn, "q", q, N, es)) || (rc = check_out(fn, "qd", qd, N, es)) || (rc = check_out(fn, "qdd", qdd, N, es)) ||
        (rc = check_out(fn, "tau", tau, N, es)))
        return rc;
    // a row of wbase is 3 pairs of reals: the kernels store it in 2-element units
    if (wrench && (rc = check_out(fn, "wbase", wbase, N, 2 * es))) return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(q);
    // the robot-specialised kernel (b2k_rne_spec.cu) serves the full 32-row tiles, the generic one the ragged tail
    const long long done = b2k_rne_spec_launch(r, wrench ? 6 /* B2K_GEN_RNE_WRENCH */ : 0 /* B2K_GEN_RNE */, dtype, q, qd, qdd, N, grav,
                                               fext, tau, wrench ? wbase : nullptr, (cudaStream_t)stream);
    if (done < 0) return (int)done;
    if (done == N) return B2K_OK;
    const size_t off = (size_t)done * r->n * es;
    if (wrench)
        return b2k_rne_wrench_launch(r, dtype, (const char *)q + off, (const char *)qd + off, (const char *)qdd + off, N - done, grav,
                                     fext, (char *)tau + off, (char *)wbase + (size_t)done * 6 * es, (cudaStream_t)stream);
    return b2k_rne_launch(r, dtype, (const char *)q + off, (const char *)qd + off, (const char *)qdd + off, N - done, grav, fext,
                          (char *)tau + off, (cudaStream_t)stream);
}

extern "C" int b2k_rne(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                       const double *grav, const double *fext, void *tau, void *stream)
{
    return rne_run("b2k_rne", r, dtype, q, qd, qdd, N, grav, fext, tau, false, nullptr, stream);
}

extern "C" int b2k_rne_wrench(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                              const double *grav, const double *fext, void *tau, void *wbase, void *stream)
{
    return rne_run("b2k_rne_wrench", r, dtype, q, qd, qdd, N, grav, fext, tau, true, wbase, stream);
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

extern "C" int b2k_fkine_jacob0_host(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *base,
                                     const double *tool, void *T, void *J, int device)
{
    const char *fn = "b2k_fkine_jacob0_host";
    int rc = check_common(fn, c, dtype, q, N, ldq, false);
    if (rc) return rc;
    if ((rc = check_out(fn, "T", T, N, 1)) || (rc = check_out(fn, "J", J, N, 1))) return rc;
    if (N == 0) return B2K_OK;
    const size_t es = dtype == B2K_F64 ? 8 : 4;
    const void *h_in[1] = {q};
    size_t in_b[1] = {(size_t)ldq * es};
    void *h_out[2] = {T, J};
    size_t out_b[2] = {16 * es, (size_t)6 * c->n * es};
    return run_pipeline(device, N, 1, h_in, in_b, 2, h_out, out_b, [&](Slot &s, long long rows) {
        return b2k_fkine_jacob0(c, dtype, s.d_in[0], rows, ldq, base, tool, s.d_out[0], s.d_out[1], s.st);
    });
}

extern "C" int b2k_fkine_host(b2k_chain_t c, int dtype, const void *q, int64_t N, int64_t ldq, const double *base,
                              const double *tool, void *T, int device)
{
    const char *fn = "b2k_fkine_host";
    int rc = check_common(fn, c, dtype, q, N, ldq, false);
    if (rc) return rc;
    if ((rc = check_out(fn, "T", T, N, 1))) return rc;
    if (N == 0) return B2K_OK;
    const size_t es = dtype == B2K_F64 ? 8 : 4;
    const void *h_in[1] = {q};
    size_t in_b[1] = {(size_t)ldq * es};
    void *h_out[1] = {T};
    size_t out_b[1] = {16 * es};
    return run_pipeline(device, N, 1, h_in, in_b, 1, h_out, out_b, [&](Slot &s, long long rows) {
        return b2k_fkine(c, dtype, s.d_in[0], rows, ldq, base, tool, s.d_out[0], s.st);
    });
}

extern "C" int b2k_rne_host(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                            const double *grav, const double *fext, void *tau, int device)
{
    const char *fn = "b2k_rne_host";
    if (!r) { b2k_set_error("%s: rne handle is NULL", fn); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (N < 0 || (N > 0 && (!q || !qd || !qdd || !tau || !grav))) { b2k_set_error("%s: NULL argument", fn); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    const size_t es = dtype == B2K_F64 ? 8 : 4;
    const void *h_in[3] = {q, qd, qdd};
    size_t in_b[3] = {r->n * es, r->n * es, r->n * es};
    void *h_out[1] = {tau};
    size_t out_b[1] = {r->n * es};
    return run_pipeline(device, N, 3, h_in, in_b, 1, h_out, out_b, [&](Slot &s, long long rows) {
        return b2k_rne(r, dtype, s.d_in[0], s.d_in[1], s.d_in[2], rows, grav, fext, s.d_out[0], s.st);
    });
}

extern "C" int b2k_rne_wrench_host(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *qdd, int64_t N,
                                   const double *grav, const double *fext, void *tau, void *wbase, int device)
{
    const char *fn = "b2k_rne_wrench_host";
    if (!r) { b2k_set_error("%s: rne handle is NULL", fn); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: bad dtype", fn); return B2K_ERR_INVALID; }
    if (N < 0 || (N > 0 && (!q || !qd || !qdd || !tau || !grav))) { b2k_set_error("%s: NULL argument", fn); return B2K_ERR_INVALID; }
    const size_t es = dtype == B2K_F64 ? 8 : 4;
    int rc;
    if ((rc = check_out(fn, "wbase", wbase, N, (unsigned)es))) return rc;
    if (N == 0) return B2K_OK;
    const void *h_in[3] = {q, qd, qdd};
    size_t in_b[3] = {r->n * es, r->n * es, r->n * es};
    void *h_out[2] = {tau, wbase};
    size_t out_b[2] = {r->n * es, 6 * es};
    return run_pipeline(device, N, 3, h_in, in_b, 2, h_out, out_b, [&](Slot &s, long long rows) {
        return b2k_rne_wrench(r, dtype, s.d_in[0], s.d_in[1], s.d_in[2], rows, grav, fext, s.d_out[0], s.d_out[1], s.st);
    });
}

// ------------------------------------------------------------------ inverse kinematics
int b2k_ik_launch_f32(const b2k_chain_s *, const void *, long long, const void *, int, int, double, int, const double *,
                      double, int, unsigned long long, int, int, void *, int *, int *, int *, void *, cudaStream_t);
int b2k_ik_launch_f64(const b2k_chain_s *, const void *, long long, const void *, int, int, double, int, const double *,
                      double, int, unsigned long long, int, int, void *, int *, int *, int *, void *, cudaStream_t);

int b2k_ik_nr_launch_f32(const b2k_chain_s *, const void *, long long, const void *, int, int, double, int, const double *,
                         double, int, unsigned long long, int, int, void *, int *, int *, int *, void *, cudaStream_t);
int b2k_ik_nr_launch_f64(const b2k_chain_s *, const void *, long long, const void *, int, int, double, int, const double *,
                         double, int, unsigned long long, int, int, void *, int *, int *, int *, void *, cudaStream_t);

extern "C" int b2k_ik_lm(b2k_chain_t c, int dtype, const void *Tep, int64_t N, const void *q0, int ilimit, int slimit,
                         double tol, int reject_jl, const double *we, double lambda, int method, uint64_t seed,
                         int semantics, int rng_per_row, void *q_out, int32_t *success, int32_t *iterations,
                         int32_t *searches, void *residual, void *stream)
{
    const char *fn = "b2k_ik_lm";
    if (!c) { b2k_set_error("%s: chain handle is NULL", fn); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: N is negative", fn); return B2K_ERR_INVALID; }
    // The solver works on the chain's own joint vector (q0 and q_out hold the n joints in chain order, i.e.
    // q[ets.jindices] -- what IKSolver.solve hands back, IK.py:216-240,346); a sub-chain of a larger robot
    // (jindices 3..6, say) is therefore served as it is.  Two joints driven by one coordinate are not.
    if (!c->distinct_jindex) {
        b2k_set_error("%s: two joints of the chain share a jindex (coupled joints are outside the solver's model)", fn);
        return B2K_ERR_INVALID;
    }
    if (ilimit < 1 || slimit < 1) { b2k_set_error("%s: ilimit and slimit must be >= 1", fn); return B2K_ERR_INVALID; }
    if (method < B2K_LM_CHAN || method > B2K_IK_GN) { b2k_set_error("%s: bad method %d", fn, method); return B2K_ERR_INVALID; }
    if (semantics != B2K_IK_SEM_CPP && semantics != B2K_IK_SEM_PYTHON) { b2k_set_error("%s: bad semantics %d", fn, semantics); return B2K_ERR_INVALID; }
    int rc;
    if ((rc = check_out(fn, "Tep", Tep, N)) || (rc = check_out(fn, "q_out", q_out, N)) ||
        (rc = check_out(fn, "success", success, N)) || (rc = check_out(fn, "iterations", iterations, N)) ||
        (rc = check_out(fn, "searches", searches, N)) || (rc = check_out(fn, "residual", residual, N)))
        return rc;
    if ((method == B2K_IK_NR || method == B2K_IK_GN) && lambda < 0) { b2k_set_error("%s: pinv_damping is negative", fn); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(Tep);
    cudaStream_t st = (cudaStream_t)stream;
    if (method == B2K_IK_NR || method == B2K_IK_GN) {
        auto nr = dtype == B2K_F64 ? b2k_ik_nr_launch_f64 : b2k_ik_nr_launch_f32;
        return nr(c, Tep, N, q0, ilimit, slimit, tol, reject_jl, we, method == B2K_IK_GN ? 0.0 : lambda, method, seed,
                  semantics, rng_per_row, q_out, success, iterations, searches, residual, st);
    }
    if (dtype == B2K_F64)
        return b2k_ik_launch_f64(c, Tep, N, q0, ilimit, slimit, tol, reject_jl, we, lambda, method, seed, semantics,
                                 rng_per_row, q_out, success, iterations, searches, residual, st);
    return b2k_ik_launch_f32(c, Tep, N, q0, ilimit, slimit, tol, reject_jl, we, lambda, method, seed, semantics,
                             rng_per_row, q_out, success, iterations, searches, residual, st);
}

int b2k_ik_ns_launch_f32(const b2k_chain_s *, const void *, long long, const void *, int, int, double, int, const double *,
                         double, int, unsigned long long, int, void *, int *, int *, int *, void *, const IkNullArgs &,
                         cudaStream_t);
int b2k_ik_ns_launch_f64(const b2k_chain_s *, const void *, long long, const void *, int, int, double, int, const double *,
                         double, int, unsigned long long, int, void *, int *, int *, int *, void *, const IkNullArgs &,
                         cudaStream_t);

extern "C" int b2k_ikine_null(b2k_chain_t c, int dtype, const void *Tep, int64_t N, const void *q0, int ilimit,
                              int slimit, double tol, int reject_jl, const double *we, double lambda, int method,
                              uint64_t seed, int rng_per_row, double kq, double km, double ps, const double *pi,
                              void *q_out, int32_t *success, int32_t *iterations, int32_t *searches, void *residual,
                              void *stream)
{
    const char *fn = "b2k_ikine_null";
    if (!c) { b2k_set_error("%s: chain handle is NULL", fn); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: N is negative", fn); return B2K_ERR_INVALID; }
    if (!c->distinct_jindex) {
        b2k_set_error("%s: two joints of the chain share a jindex (coupled joints are outside the solver's model)", fn);
        return B2K_ERR_INVALID;
    }
    if (c->n < 7 || c->n > B2K_MAX_JOINTS) {
        b2k_set_error("%s: the null-space terms need a redundant chain of 7..%d joints (n = %d)", fn, B2K_MAX_JOINTS, c->n);
        return B2K_ERR_INVALID;
    }
    if (ilimit < 1 || slimit < 1) { b2k_set_error("%s: ilimit and slimit must be >= 1", fn); return B2K_ERR_INVALID; }
    if (method < B2K_LM_CHAN || method > B2K_IK_GN) { b2k_set_error("%s: bad method %d", fn, method); return B2K_ERR_INVALID; }
    if (!isfinite(kq) || !isfinite(km)) { b2k_set_error("%s: kq and km must be finite", fn); return B2K_ERR_INVALID; }
    if (!(kq > 0) && !(km > 0)) { b2k_set_error("%s: at least one of kq and km must be > 0", fn); return B2K_ERR_INVALID; }
    if (!isfinite(ps)) { b2k_set_error("%s: ps must be finite", fn); return B2K_ERR_INVALID; }
    if (!pi) { b2k_set_error("%s: pi is NULL", fn); return B2K_ERR_INVALID; }
    for (int i = 0; i < c->n; i++) {
        if (!isfinite(pi[i])) { b2k_set_error("%s: pi[%d] is not finite", fn, i); return B2K_ERR_INVALID; }
        if (kq > 0 && ps == pi[i]) { b2k_set_error("%s: ps == pi[%d] divides by zero in the joint-limit term", fn, i); return B2K_ERR_INVALID; }
    }
    int rc;
    if ((rc = check_out(fn, "Tep", Tep, N)) || (rc = check_out(fn, "q_out", q_out, N)) ||
        (rc = check_out(fn, "success", success, N)) || (rc = check_out(fn, "iterations", iterations, N)) ||
        (rc = check_out(fn, "searches", searches, N)) || (rc = check_out(fn, "residual", residual, N)))
        return rc;
    if ((method == B2K_IK_NR || method == B2K_IK_GN) && lambda < 0) { b2k_set_error("%s: pinv_damping is negative", fn); return B2K_ERR_INVALID; }
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(Tep);
    const IkNullArgs ns{kq, km, ps, pi};
    auto launch = dtype == B2K_F64 ? b2k_ik_ns_launch_f64 : b2k_ik_ns_launch_f32;
    return launch(c, Tep, N, q0, ilimit, slimit, tol, reject_jl, we, method == B2K_IK_GN ? 0.0 : lambda, method, seed,
                  rng_per_row, q_out, success, iterations, searches, residual, ns, (cudaStream_t)stream);
}

// ------------------------------------------------------------------ dynamics fan-outs
int b2k_rne_fan_launch_f32(const b2k_rne_s *, int, const void *, const void *, const void *, long long, const double *, void *, cudaStream_t);
int b2k_rne_fan_launch_f64(const b2k_rne_s *, int, const void *, const void *, const void *, long long, const double *, void *, cudaStream_t);
enum { FAN_INERTIA = 0, FAN_GRAVLOAD = 1, FAN_ITORQUE = 2, FAN_CORIOLIS = 3, FAN_ACCEL = 4 };

static int fan_dispatch(const char *fn, b2k_rne_t r, int dtype, int mode, const void *in0, const void *in1, const void *in2,
                        int nin, int64_t N, const double *grav, bool need_grav, void *out, void *stream)
{
    if (!r) { b2k_set_error("%s: rne handle is NULL", fn); return B2K_ERR_INVALID; }
    if (dtype != B2K_F32 && dtype != B2K_F64) { b2k_set_error("%s: dtype must be B2K_F32 or B2K_F64", fn); return B2K_ERR_INVALID; }
    if (N < 0) { b2k_set_error("%s: N is negative", fn); return B2K_ERR_INVALID; }
    if (need_grav && !grav) { b2k_set_error("%s: grav is NULL (pass -robot.gravity like DHRobot.rne)", fn); return B2K_ERR_INVALID; }
    int rc;
    const unsigned es = dtype == B2K_F64 ? 8u : 4u;
    if ((rc = check_out(fn, "q", in0, N, es)) || (nin >= 2 && (rc = check_out(fn, "second input", in1, N, es))) ||
        (nin >= 3 && (rc = check_out(fn, "third input", in2, N, es))) || (rc = check_out(fn, "output", out, N, es)))
        return rc;
    if (N == 0) return B2K_OK;
    B2K_ON_DEVICE_OF(in0);
    cudaStream_t st = (cudaStream_t)stream;
    const long long done = b2k_rne_spec_launch(r, mode + 1 /* FAN_* -> B2K_GEN_* */, dtype, in0, in1, in2, N, grav, nullptr, out, nullptr, st);
    if (done < 0) return (int)done;
    if (done == N) return B2K_OK;
    const size_t off = (size_t)done * r->n * es;
    const size_t out_per_row = (mode == FAN_INERTIA || mode == FAN_CORIOLIS) ? (size_t)r->n * r->n : (size_t)r->n;
    in0 = (const char *)in0 + off;
    if (in1) in1 = (const char *)in1 + off;
    if (in2) in2 = (const char *)in2 + off;
    out = (char *)out + (size_t)done * out_per_row * es;
    N -= done;
    if (dtype == B2K_F64) return b2k_rne_fan_launch_f64(r, mode, in0, in1, in2, N, grav, out, st);
    return b2k_rne_fan_launch_f32(r, mode, in0, in1, in2, N, grav, out, st);
}

extern "C" int b2k_rne_inertia(b2k_rne_t r, int dtype, const void *q, int64_t N, void *M, void *stream)
{
    return fan_dispatch("b2k_rne_inertia", r, dtype, FAN_INERTIA, q, nullptr, nullptr, 1, N, nullptr, false, M, stream);
}
extern "C" int b2k_rne_gravload(b2k_rne_t r, int dtype, const void *q, int64_t N, const double *grav, void *taug, void *stream)
{
    return fan_dispatch("b2k_rne_gravload", r, dtype, FAN_GRAVLOAD, q, nullptr, nullptr, 1, N, grav, true, taug, stream);
}
extern "C" int b2k_rne_itorque(b2k_rne_t r, int dtype, const void *q, const void *qdd, int64_t N, void *taui, void *stream)
{
    return fan_dispatch("b2k_rne_itorque", r, dtype, FAN_ITORQUE, q, qdd, nullptr, 2, N, nullptr, false, taui, stream);
}
extern "C" int b2k_rne_coriolis(b2k_rne_t r, int dtype, const void *q, const void *qd, int64_t N, void *Cm, void *stream)
{
    return fan_dispatch("b2k_rne_coriolis", r, dtype, FAN_CORIOLIS, q, qd, nullptr, 2, N, nullptr, false, Cm, stream);
}
extern "C" int b2k_rne_accel(b2k_rne_t r, int dtype, const void *q, const void *qd, const void *torque, int64_t N,
                             const double *grav, void *qdd, void *stream)
{
    return fan_dispatch("b2k_rne_accel", r, dtype, FAN_ACCEL, q, qd, torque, 3, N, grav, true, qdd, stream);
}
