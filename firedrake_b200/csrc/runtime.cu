// Runtime plumbing of libfdb200: context, device memory, the host-pointer
// mirror cache, timers.  No numerics here.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <unordered_map>

#include "common.cuh"

namespace fdb {

static Context g_ctx;
static thread_local char g_err[1024] = "";

Context &ctx() { return g_ctx; }

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int require_init()
{
    if (!g_ctx.ready) {
        set_error("fdb_init() has not been called");
        return 1;
    }
    return 0;
}

struct Mirror {
    void *dev = nullptr;
    size_t nbytes = 0;
    uint64_t version = 0;
    bool valid = false;
    uint64_t epoch = 0;      // last fdb_kernel_call that touched it (LRU eviction)
};
static std::unordered_map<const void *, Mirror> g_mirrors;
// The cache is bounded: when the mirrors exceed g_mirror_limit bytes, the least recently used
// ones that the CURRENT call has not touched are released (a time loop over fresh host buffers
// would otherwise grow without bound).  FDB_MIRROR_LIMIT_MB overrides (default: 60 % of HBM).
static size_t g_mirror_bytes = 0, g_mirror_limit = 0;
static uint64_t g_epoch = 1;

}  // namespace fdb

using namespace fdb;

int fdb_opt_matrix_kernel = getenv("FDB_MATRIX_DMMA") ? atoi(getenv("FDB_MATRIX_DMMA")) : -1;

static cudaStream_t g_side = nullptr;
static cudaEvent_t g_side_ev = nullptr, g_main_ev = nullptr;
static bool g_side_pending = false;

void fdb_mirror_new_epoch() { fdb::g_epoch++; }

bool fdb_mirror_is_current(const void *host, size_t nbytes, uint64_t version)
{
    auto it = fdb::g_mirrors.find(host);
    return it != fdb::g_mirrors.end() && it->second.valid && it->second.nbytes == nbytes &&
           it->second.version == version;
}

extern "C" {

const char *fdb_last_error(void) { return g_err; }

int fdb_init(int device)
{
    Context &c = ctx();
    if (c.ready) {
        if (c.device != device) {
            set_error("fdb_init: already initialised on device %d", c.device);
            return 1;
        }
        return 0;
    }
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        set_error("fdb_init: no CUDA device available (%s)", cudaGetErrorString(e));
        return 1;
    }
    if (device < 0 || device >= n) {
        set_error("fdb_init: device %d out of range (have %d)", device, n);
        return 1;
    }
    FDB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    FDB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_error("fdb_init: device %s is sm_%d%d; this library is built for sm_90a only",
                  prop.name, prop.major, prop.minor);
        return 1;
    }
    c.device = device;
    c.sm_count = prop.multiProcessorCount;
    FDB_CUDA(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
    FDB_CUDA(cudaMalloc(&c.reduce_scratch, 4096 * sizeof(double)));
    FDB_CUDA(cudaMalloc(&c.work_counter, 64 * sizeof(int)));
    FDB_CUDA(cudaHostAlloc((void **)&c.reduce_host, 64 * sizeof(double), cudaHostAllocDefault));
    c.ready = true;
    return 0;
}

int fdb_finalize(void)
{
    Context &c = ctx();
    if (!c.ready) return 0;
    cudaStreamSynchronize(c.stream);
    for (auto &kv : g_mirrors) cudaFree(kv.second.dev);
    g_mirrors.clear();
    g_mirror_bytes = 0;
    if (c.flush_buf) cudaFree(c.flush_buf);
    if (g_side) {
        cudaStreamSynchronize(g_side);
        cudaStreamDestroy(g_side);
        cudaEventDestroy(g_side_ev);
        cudaEventDestroy(g_main_ev);
        g_side = nullptr;
        g_side_pending = false;
    }
    fdb_bv_release();
    cudaFree(c.reduce_scratch);
    cudaFree(c.work_counter);
    cudaFreeHost(c.reduce_host);
    cudaStreamDestroy(c.stream);
    c = Context();
    return 0;
}

int fdb_synchronize(void)
{
    if (require_init()) return 1;
    FDB_CUDA(cudaStreamSynchronize(ctx().stream));
    return 0;
}

int fdb_device_info(char *name, int name_len, int *sm_count, size_t *total_mem)
{
    if (require_init()) return 1;
    cudaDeviceProp prop;
    FDB_CUDA(cudaGetDeviceProperties(&prop, ctx().device));
    if (name && name_len > 0) {
        strncpy(name, prop.name, name_len - 1);
        name[name_len - 1] = 0;
    }
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (total_mem) *total_mem = prop.totalGlobalMem;
    return 0;
}

uint64_t fdb_launch_count(void) { return ctx().launches; }

static int *option_slot(const char *name)
{
    if (name && !strcmp(name, "matrix_kernel")) return &fdb_opt_matrix_kernel;
    return nullptr;
}

int fdb_set_option(const char *name, int value)
{
    int *s = option_slot(name);
    if (!s) {
        set_error("fdb_set_option: unknown option '%s'", name ? name : "(null)");
        return 1;
    }
    *s = value;
    return 0;
}

int fdb_get_option(const char *name, int *value)
{
    int *s = option_slot(name);
    if (!s) {
        set_error("fdb_get_option: unknown option '%s'", name ? name : "(null)");
        return 1;
    }
    *value = *s;
    return 0;
}

void *fdb_malloc(size_t nbytes)
{
    if (require_init()) return nullptr;
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, nbytes ? nbytes : 1);
    if (e != cudaSuccess) {
        set_error("fdb_malloc(%zu): %s", nbytes, cudaGetErrorString(e));
        return nullptr;
    }
    return p;
}

int fdb_free(void *dptr)
{
    if (require_init()) return 1;
    if (g_side) FDB_CUDA(cudaStreamSynchronize(g_side));
    FDB_CUDA(cudaStreamSynchronize(ctx().stream));
    FDB_CUDA(cudaFree(dptr));
    return 0;
}

int fdb_memset(void *dptr, int value, size_t nbytes)
{
    if (require_init()) return 1;
    FDB_CUDA(cudaMemsetAsync(dptr, value, nbytes, ctx().stream));
    return 0;
}

int fdb_memcpy_h2d(void *dst, const void *src, size_t nbytes)
{
    if (require_init()) return 1;
    FDB_CUDA(cudaMemcpyAsync(dst, src, nbytes, cudaMemcpyHostToDevice, ctx().stream));
    FDB_CUDA(cudaStreamSynchronize(ctx().stream));
    return 0;
}

int fdb_memcpy_d2h(void *dst, const void *src, size_t nbytes)
{
    if (require_init()) return 1;
    FDB_CUDA(cudaMemcpyAsync(dst, src, nbytes, cudaMemcpyDeviceToHost, ctx().stream));
    FDB_CUDA(cudaStreamSynchronize(ctx().stream));
    return 0;
}

int fdb_memcpy_d2d(void *dst, const void *src, size_t nbytes)
{
    if (require_init()) return 1;
    FDB_CUDA(cudaMemcpyAsync(dst, src, nbytes, cudaMemcpyDeviceToDevice, ctx().stream));
    return 0;
}

// A deliberately narrow zeroing kernel: a full-speed cudaMemset saturates HBM and
// stalls the (compute-bound, but latency-sensitive) global kernel it overlaps for
// exactly its own duration; a few CTAs trickle the zeros out over the whole
// kernel instead.
__global__ void __launch_bounds__(256) k_zero_trickle(uint4 *p, size_t n16)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const uint4 z = make_uint4(0, 0, 0, 0);
    for (; i < n16; i += stride) p[i] = z;
}

int fdb_zero_background(void *dptr, size_t nbytes)
{
    if (require_init()) return 1;
    if (!g_side) {
        FDB_CUDA(cudaStreamCreateWithFlags(&g_side, cudaStreamNonBlocking));
        FDB_CUDA(cudaEventCreateWithFlags(&g_side_ev, cudaEventDisableTiming));
        FDB_CUDA(cudaEventCreateWithFlags(&g_main_ev, cudaEventDisableTiming));
    }
    FDB_CUDA(cudaEventRecord(g_main_ev, ctx().stream));
    FDB_CUDA(cudaStreamWaitEvent(g_side, g_main_ev, 0));
    static const int nblk = getenv("FDB_ZERO_CTAS") ? atoi(getenv("FDB_ZERO_CTAS")) : 0;
    const size_t n16 = nbytes / 16;
    if (nblk > 0 && n16 > 0) {
        k_zero_trickle<<<nblk, 256, 0, g_side>>>((uint4 *)dptr, n16);
        FDB_LAUNCH_CHECK();
        if (nbytes % 16)
            FDB_CUDA(cudaMemsetAsync((char *)dptr + n16 * 16, 0, nbytes % 16, g_side));
    } else {
        FDB_CUDA(cudaMemsetAsync(dptr, 0, nbytes, g_side));
    }
    FDB_CUDA(cudaEventRecord(g_side_ev, g_side));
    g_side_pending = true;
    return 0;
}

int fdb_background_barrier(void)
{
    if (require_init()) return 1;
    if (g_side_pending) {
        FDB_CUDA(cudaStreamWaitEvent(ctx().stream, g_side_ev, 0));
        g_side_pending = false;
    }
    return 0;
}

void *fdb_host_alloc(size_t nbytes)
{
    if (require_init()) return nullptr;
    void *p = nullptr;
    cudaError_t e = cudaHostAlloc(&p, nbytes ? nbytes : 1, cudaHostAllocDefault);
    if (e != cudaSuccess) {
        set_error("fdb_host_alloc(%zu): %s", nbytes, cudaGetErrorString(e));
        return nullptr;
    }
    return p;
}

int fdb_host_free(void *hptr)
{
    if (require_init()) return 1;
    FDB_CUDA(cudaFreeHost(hptr));
    return 0;
}

int fdb_host_register(void *hptr, size_t nbytes)
{
    if (require_init()) return 1;
    FDB_CUDA(cudaHostRegister(hptr, nbytes, cudaHostRegisterDefault));
    return 0;
}

int fdb_host_unregister(void *hptr)
{
    if (require_init()) return 1;
    FDB_CUDA(cudaHostUnregister(hptr));
    return 0;
}

/* ---------------------------------------------------------------- mirror cache */

int fdb_mirror_acquire(const void *host, size_t nbytes, uint64_t version, int upload,
                       void **dev_out)
{
    if (require_init()) return 1;
    if (!host) {
        set_error("fdb_mirror_acquire: NULL host pointer");
        return 1;
    }
    Mirror &m = g_mirrors[host];
    if (m.dev && m.nbytes != nbytes) {
        FDB_CUDA(cudaStreamSynchronize(ctx().stream));
        FDB_CUDA(cudaFree(m.dev));
        g_mirror_bytes -= m.nbytes;
        m = Mirror();
    }
    m.epoch = g_epoch;
    if (!m.dev) {
        if (!g_mirror_limit) {
            const char *e = getenv("FDB_MIRROR_LIMIT_MB");
            size_t fr = 0, tot = 0;
            cudaMemGetInfo(&fr, &tot);
            g_mirror_limit = e ? (size_t)atoll(e) << 20 : (size_t)(0.6 * (double)tot);
        }
        while (g_mirror_bytes + nbytes > g_mirror_limit) {
            auto victim = g_mirrors.end();
            for (auto it = g_mirrors.begin(); it != g_mirrors.end(); ++it)
                if (it->second.dev && it->second.epoch != g_epoch &&
                    (victim == g_mirrors.end() || it->second.epoch < victim->second.epoch))
                    victim = it;
            if (victim == g_mirrors.end()) break;      // everything left is in use by this call
            FDB_CUDA(cudaStreamSynchronize(ctx().stream));
            FDB_CUDA(cudaFree(victim->second.dev));
            g_mirror_bytes -= victim->second.nbytes;
            g_mirrors.erase(victim);                   // (rehash-safe: `m` is re-looked-up below)
        }
        Mirror &mm = g_mirrors[host];
        FDB_CUDA(cudaMalloc(&mm.dev, nbytes ? nbytes : 1));
        mm.nbytes = nbytes;
        mm.valid = false;
        mm.epoch = g_epoch;
        g_mirror_bytes += nbytes;
        if (upload) {
            FDB_CUDA(cudaMemcpyAsync(mm.dev, host, nbytes, cudaMemcpyHostToDevice, ctx().stream));
            mm.valid = true;
            mm.version = version;
        }
        *dev_out = mm.dev;
        return 0;
    }
    if (upload && (!m.valid || m.version != version)) {
        FDB_CUDA(cudaMemcpyAsync(m.dev, host, nbytes, cudaMemcpyHostToDevice, ctx().stream));
        m.valid = true;
        m.version = version;
    }
    *dev_out = m.dev;
    return 0;
}

int fdb_mirror_writeback(void *host)
{
    if (require_init()) return 1;
    auto it = g_mirrors.find(host);
    if (it == g_mirrors.end()) {
        set_error("fdb_mirror_writeback: %p has no mirror", host);
        return 1;
    }
    FDB_CUDA(cudaMemcpyAsync(host, it->second.dev, it->second.nbytes, cudaMemcpyDeviceToHost,
                             ctx().stream));
    FDB_CUDA(cudaStreamSynchronize(ctx().stream));
    return 0;
}

int fdb_mirror_set_version(const void *host, uint64_t version)
{
    auto it = g_mirrors.find(host);
    if (it == g_mirrors.end()) return 1;
    it->second.version = version;
    it->second.valid = true;
    return 0;
}

// Partial transfers between a host buffer and its mirror (the partitioned host path of
// op2.Parloop: rows the chunked pipeline did not move).  Asynchronous on the engine stream;
// `sync` waits for the download before returning.
int fdb_mirror_upload_range(const void *host, size_t offset, size_t nbytes)
{
    if (require_init()) return 1;
    auto it = g_mirrors.find(host);
    if (it == g_mirrors.end() || offset + nbytes > it->second.nbytes) {
        set_error("fdb_mirror_upload_range: %p has no mirror of at least %zu bytes", host, offset + nbytes);
        return 1;
    }
    if (nbytes)
        FDB_CUDA(cudaMemcpyAsync((char *)it->second.dev + offset, (const char *)host + offset, nbytes,
                                 cudaMemcpyHostToDevice, ctx().stream));
    return 0;
}

int fdb_mirror_download_range(void *host, size_t offset, size_t nbytes, int sync)
{
    if (require_init()) return 1;
    auto it = g_mirrors.find(host);
    if (it == g_mirrors.end() || offset + nbytes > it->second.nbytes) {
        set_error("fdb_mirror_download_range: %p has no mirror of at least %zu bytes", host, offset + nbytes);
        return 1;
    }
    if (nbytes)
        FDB_CUDA(cudaMemcpyAsync((char *)host + offset, (const char *)it->second.dev + offset, nbytes,
                                 cudaMemcpyDeviceToHost, ctx().stream));
    if (sync) FDB_CUDA(cudaStreamSynchronize(ctx().stream));
    return 0;
}

int fdb_mirror_drop(const void *host)
{
    if (require_init()) return 1;
    auto it = g_mirrors.find(host);
    if (it == g_mirrors.end()) return 0;
    FDB_CUDA(cudaStreamSynchronize(ctx().stream));
    FDB_CUDA(cudaFree(it->second.dev));
    g_mirror_bytes -= it->second.nbytes;
    g_mirrors.erase(it);
    return 0;
}

int fdb_mirror_drop_all(void)
{
    if (require_init()) return 1;
    FDB_CUDA(cudaStreamSynchronize(ctx().stream));
    for (auto &kv : g_mirrors) cudaFree(kv.second.dev);
    g_mirrors.clear();
    g_mirror_bytes = 0;
    return 0;
}

/* ---------------------------------------------------------------------- timers */

struct fdb_timer_s {
    cudaEvent_t a, b;
};

int fdb_timer_create(fdb_timer_t *out)
{
    if (require_init()) return 1;
    fdb_timer_s *t = new fdb_timer_s;
    FDB_CUDA(cudaEventCreate(&t->a));
    FDB_CUDA(cudaEventCreate(&t->b));
    *out = t;
    return 0;
}

int fdb_timer_start(fdb_timer_t t)
{
    FDB_CUDA(cudaEventRecord(t->a, ctx().stream));
    return 0;
}

int fdb_timer_stop(fdb_timer_t t, float *ms_out)
{
    FDB_CUDA(cudaEventRecord(t->b, ctx().stream));
    FDB_CUDA(cudaEventSynchronize(t->b));
    FDB_CUDA(cudaEventElapsedTime(ms_out, t->a, t->b));
    return 0;
}

int fdb_timer_destroy(fdb_timer_t t)
{
    cudaEventDestroy(t->a);
    cudaEventDestroy(t->b);
    delete t;
    return 0;
}

int fdb_flush_l2(void)
{
    if (require_init()) return 1;
    Context &c = ctx();
    if (!c.flush_buf) {
        c.flush_bytes = (size_t)128 << 20;   // more than 2x the 50 MB L2 of an H100
        FDB_CUDA(cudaMalloc(&c.flush_buf, c.flush_bytes));
    }
    FDB_CUDA(cudaMemsetAsync(c.flush_buf, 0, c.flush_bytes, c.stream));
    return 0;
}

}  // extern "C"
