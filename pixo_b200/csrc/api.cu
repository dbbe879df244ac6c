// api.cu — the extern "C" surface of libpixo_b200.so (see include/pixo_b200.h): errors, scratch buffers, the host
// pool, the staging copies and the one staging path of the host-buffer entry points, and the context and memory
// entry points.  The format entry points are in api_jpeg.cu, api_png.cu and api_decode.cu.
#include <stdarg.h>
#include <string.h>

#include <emmintrin.h>

#include <algorithm>
#include <thread>
#include <vector>

#include "api.hpp"

namespace pixo {

static thread_local std::string g_thread_err;

int set_error(pixo_b200_ctx *ctx, int code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (ctx) ctx->err = buf;
    g_thread_err = buf;
    return code;
}

int cuda_fail(pixo_b200_ctx *ctx, cudaError_t e, const char *what)
{
    const int code = e == cudaErrorMemoryAllocation ? PIXO_B200_ERR_OOM : PIXO_B200_ERR_CUDA;
    return set_error(ctx, code, "CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
}

template <bool Pinned>
int Buffer<Pinned>::ensure(pixo_b200_ctx *ctx, size_t bytes)
{
    if (cap >= bytes) return 0;
    if (ptr) {
        PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if constexpr (Pinned) PIXO_CUDA(ctx, cudaFreeHost(ptr));
        else PIXO_CUDA(ctx, cudaFree(ptr));
        ptr = nullptr;
        cap = 0;
    }
    const size_t want = bytes + bytes / 8 + 256;
    if constexpr (Pinned) PIXO_CUDA(ctx, cudaMallocHost(&ptr, want));
    else PIXO_CUDA(ctx, cudaMalloc(&ptr, want));
    cap = want;
    return 0;
}

template struct Buffer<false>;
template struct Buffer<true>;

HostPool::HostPool(int nthreads)
{
    for (int i = 0; i < nthreads; ++i) threads_.emplace_back([this] { worker(); });
}

HostPool::~HostPool()
{
    {
        std::lock_guard<std::mutex> lk(m_);
        stop_ = true;
    }
    cv_work_.notify_all();
    for (auto &t : threads_) t.join();
}

void HostPool::worker()
{
    uint64_t seen = 0;
    for (;;) {
        const std::function<void(int)> *fn;
        int n;
        {
            std::unique_lock<std::mutex> lk(m_);
            cv_work_.wait(lk, [&] { return stop_ || generation_ != seen; });
            if (stop_) return;
            seen = generation_;
            fn = fn_;
            n = njobs_;
            // woke after that run() had returned: claiming from next_ now would take a job of the next run()
            if (!fn) continue;
            ++active_;
        }
        for (int j; (j = next_.fetch_add(1)) < n;) (*fn)(j);
        {
            std::lock_guard<std::mutex> lk(m_);
            if (--active_ == 0) cv_done_.notify_all();
        }
    }
}

void HostPool::run(int njobs, const std::function<void(int)> &fn)
{
    if (njobs <= 0) return;
    {
        std::lock_guard<std::mutex> lk(m_);
        fn_ = &fn;
        njobs_ = njobs;
        next_.store(0);
        ++generation_;
    }
    if (njobs > 1) cv_work_.notify_all();
    for (int j; (j = next_.fetch_add(1)) < njobs;) fn(j);
    // every job has been claimed; wait for the workers that are still inside one (a worker that
    // wakes up late finds nothing to claim and leaves at once)
    std::unique_lock<std::mutex> lk(m_);
    cv_done_.wait(lk, [&] { return active_ == 0; });
    fn_ = nullptr;
    njobs_ = 0;
}

static HostPool *host_pool(pixo_b200_ctx *ctx)
{
    if (!ctx->pool) {
        int n = ctx->host_threads - 1;
        n = n < 1 ? 1 : (n > 5 ? 5 : n);   // five helpers + the caller saturate a socket's copy bandwidth
        ctx->pool = std::make_unique<HostPool>(n);
    }
    return ctx->pool.get();
}

// Copy into a pinned staging slot with NON-TEMPORAL stores.  An ordinary memcpy of a 1 MB piece
// leaves the bytes dirty in the copying core's cache, and the DMA engine then has to pull every
// line out of that cache; streaming stores
// go to memory and the DMA reads it at the pinned rate.
static void stage_copy(void *dst, const void *src, size_t n)
{
#if defined(__x86_64__) || defined(__SSE2__)
    auto *d = reinterpret_cast<uint8_t *>(dst);
    auto *s = reinterpret_cast<const uint8_t *>(src);
    if ((reinterpret_cast<uintptr_t>(d) & 15) == 0) {
        size_t i = 0;
        for (; i + 64 <= n; i += 64) {
            const __m128i a = _mm_loadu_si128(reinterpret_cast<const __m128i *>(s + i));
            const __m128i b = _mm_loadu_si128(reinterpret_cast<const __m128i *>(s + i + 16));
            const __m128i c = _mm_loadu_si128(reinterpret_cast<const __m128i *>(s + i + 32));
            const __m128i e = _mm_loadu_si128(reinterpret_cast<const __m128i *>(s + i + 48));
            _mm_stream_si128(reinterpret_cast<__m128i *>(d + i), a);
            _mm_stream_si128(reinterpret_cast<__m128i *>(d + i + 16), b);
            _mm_stream_si128(reinterpret_cast<__m128i *>(d + i + 32), c);
            _mm_stream_si128(reinterpret_cast<__m128i *>(d + i + 48), e);
        }
        _mm_sfence();
        if (i < n) memcpy(d + i, s + i, n - i);
        return;
    }
#endif
    memcpy(dst, src, n);
}

bool is_page_locked(const void *p)
{
    cudaPointerAttributes at;
    const bool locked = cudaPointerGetAttributes(&at, p) == cudaSuccess &&
                        (at.type == cudaMemoryTypeHost || at.type == cudaMemoryTypeManaged);
    cudaGetLastError();  // an unregistered pointer is not an error here
    return locked;
}

// Host -> device copy that does not depend on the caller's buffer being page-locked.  pixo's
// callers hand over ordinary (pageable) memory, and the driver's own pageable path moves it through
// one staging thread.  Here the context's host threads copy 1 MB pieces into a ring of
// pinned slots and each queues the DMA of its piece as soon as it is staged, so the host copies run
// in parallel with each other and with the DMA engine, and the link runs near its pinned rate
// (see DESIGN.md section 5).
// Page-locked sources, and small ones, go straight to cudaMemcpyAsync.
int h2d_copy(pixo_b200_ctx *ctx, void *dst, const void *src, size_t bytes, cudaStream_t st)
{
    constexpr size_t SLOT = (size_t)1 << 20;
    constexpr int NSLOT = 32;
    if (bytes < 4 * SLOT || is_page_locked(src)) {
        PIXO_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st));
        return 0;
    }
    PIXO_TRY(ctx->h_in.ensure(ctx, SLOT * NSLOT));
    while (ctx->stage_events.size() < (size_t)NSLOT) {
        cudaEvent_t ev;
        PIXO_CUDA(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        PIXO_CUDA(ctx, cudaEventRecord(ev, st));
        ctx->stage_events.push_back(ev);
    }
    const int nchunks = (int)((bytes + SLOT - 1) / SLOT);
    std::atomic<int> first_error{(int)cudaSuccess};
    const int device = ctx->device;
    // piece c uses slot c % NSLOT; pieces are claimed in order, so a slot's previous user is always
    // NSLOT pieces back and its DMA has normally drained long before the slot comes round again
    auto piece = [&](int c) {
        if (first_error.load() != (int)cudaSuccess) return;
        cudaError_t e = cudaSetDevice(device);
        const int slot_i = c % NSLOT;
        uint8_t *slot = ctx->h_in.slot(slot_i, SLOT);
        const size_t off = (size_t)c * SLOT, n = std::min(SLOT, bytes - off);
        if (e == cudaSuccess) e = cudaEventSynchronize(ctx->stage_events[slot_i]);   // the slot's previous DMA (this call's or the last one's) has drained
        if (e == cudaSuccess) {
            stage_copy(slot, reinterpret_cast<const uint8_t *>(src) + off, n);
            e = cudaMemcpyAsync(reinterpret_cast<uint8_t *>(dst) + off, slot, n, cudaMemcpyHostToDevice, st);
        }
        if (e == cudaSuccess && c + NSLOT < nchunks) e = cudaEventRecord(ctx->stage_events[slot_i], st);
        if (e != cudaSuccess) { int ok = (int)cudaSuccess; first_error.compare_exchange_strong(ok, (int)e); }
    };
    if (nchunks > NSLOT) {
        // a slot is reused: its event must be recorded by the piece that used it before.  Run the
        // pieces in rounds of NSLOT so that "previous user" is always in an earlier round.
        for (int r0 = 0; r0 < nchunks; r0 += NSLOT) {
            const int cnt = std::min(NSLOT, nchunks - r0);
            host_pool(ctx)->run(cnt, [&](int j) { piece(r0 + j); });
        }
    } else {
        host_pool(ctx)->run(nchunks, piece);
    }
    // the slots may be rewritten by the next call: make that call wait for this one's DMAs
    PIXO_CUDA(ctx, (cudaError_t)first_error.load());
    for (int s_i = 0; s_i < std::min(nchunks, NSLOT); ++s_i) PIXO_CUDA(ctx, cudaEventRecord(ctx->stage_events[s_i], st));
    return 0;
}

// Device -> pageable host: through the pinned ring with the pool copying out, for results big
// enough to matter (a 4K JPEG is ~3 MB).  Synchronous: returns when `dst` holds the bytes.
int d2h_copy_sync(pixo_b200_ctx *ctx, void *dst, const void *src, size_t bytes, cudaStream_t st)
{
    constexpr size_t PIECE = (size_t)512 << 10;
    if (bytes < 2 * PIECE || is_page_locked(dst)) {
        PIXO_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st));
        PIXO_CUDA(ctx, cudaStreamSynchronize(st));
        return 0;
    }
    PIXO_TRY(ctx->h_out.ensure(ctx, bytes));
    PIXO_CUDA(ctx, cudaMemcpyAsync(ctx->h_out.ptr, src, bytes, cudaMemcpyDeviceToHost, st));
    PIXO_CUDA(ctx, cudaStreamSynchronize(st));
    const int n = (int)((bytes + PIECE - 1) / PIECE);
    host_pool(ctx)->run(n, [&](int j) {
        const size_t off = (size_t)j * PIECE, len = std::min(PIECE, bytes - off);
        memcpy(reinterpret_cast<uint8_t *>(dst) + off, ctx->h_out.slot(j, PIECE), len);
    });
    return 0;
}

DrainOnError::~DrainOnError()
{
    if (!armed) return;
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(ctx->copy_stream);
    cudaStreamSynchronize(ctx->d2h_stream);
    cudaGetLastError();
}

int stage_host_call(pixo_b200_ctx *ctx, const void *in, size_t in_bytes, const std::function<void(Layout &)> &outputs,
                    const std::function<int(const uint8_t *d_in, HostResults &back)> &queue)
{
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    PIXO_TRY(ctx->d_in.ensure(ctx, in_bytes));
    PIXO_TRY(bind(ctx, ctx->d_out, outputs));
    DrainOnError drain(ctx);
    if (in_bytes) PIXO_TRY(h2d_copy(ctx, ctx->d_in.ptr, in, in_bytes, ctx->stream));
    HostResults back;
    PIXO_TRY(queue(static_cast<const uint8_t *>(ctx->d_in.ptr), back));
    for (const HostResult &r : back) {
        if (r.out_len) {
            *r.out_len = r.bytes;
            if (r.bytes > r.cap)
                return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "output capacity %zu below %zu", r.cap, r.bytes);
        }
        if (r.dst) PIXO_TRY(d2h_copy_sync(ctx, r.dst, r.src, r.bytes, ctx->stream));
    }
    drain.armed = false;
    return 0;
}

}  // namespace pixo

using namespace pixo;

pixo_b200_ctx::~pixo_b200_ctx()
{
    for (cudaEvent_t ev : stage_events) cudaEventDestroy(ev);
    for (cudaEvent_t ev : {switch_event, resize_events[0], resize_events[1], ev_in[0], ev_in[1], ev_used[0], ev_used[1],
                           ev_out[0], ev_out[1], ev_len[0], ev_len[1]})
        if (ev) cudaEventDestroy(ev);
    if (own_stream) cudaStreamDestroy(own_stream);
    if (copy_stream) cudaStreamDestroy(copy_stream);
    if (d2h_stream) cudaStreamDestroy(d2h_stream);
}

extern "C" {

int pixo_b200_version(void) { return PIXO_B200_VERSION; }

int pixo_b200_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int pixo_b200_ctx_create(int device, pixo_b200_ctx **out)
{
    if (!out) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx out pointer is null");
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        return set_error(nullptr, PIXO_B200_ERR_CUDA,
                         "no CUDA device available (%s); libpixo_b200 has no CPU fallback",
                         e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    if (device < 0 || device >= n)
        return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "device %d out of range (0..%d)", device, n - 1);
    auto ctx = std::make_unique<pixo_b200_ctx>();
    ctx->device = device;
    if ((e = cudaSetDevice(device)) != cudaSuccess) return cuda_fail(nullptr, e, "cudaSetDevice");
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return cuda_fail(nullptr, e, "cudaGetDeviceProperties");
    ctx->sm_count = prop.multiProcessorCount;
    if ((e = cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking)) != cudaSuccess ||
        (e = cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking)) != cudaSuccess ||
        (e = cudaStreamCreateWithFlags(&ctx->d2h_stream, cudaStreamNonBlocking)) != cudaSuccess)
        return cuda_fail(nullptr, e, "cudaStreamCreate");
    for (cudaEvent_t *ev : {&ctx->switch_event, &ctx->resize_events[0], &ctx->resize_events[1], &ctx->ev_in[0],
                            &ctx->ev_in[1], &ctx->ev_used[0], &ctx->ev_used[1], &ctx->ev_out[0], &ctx->ev_out[1],
                            &ctx->ev_len[0], &ctx->ev_len[1]})
        if ((e = cudaEventCreateWithFlags(ev, cudaEventDisableTiming)) != cudaSuccess)
            return cuda_fail(nullptr, e, "cudaEventCreate");
    ctx->stream = ctx->own_stream;
    unsigned hc = std::thread::hardware_concurrency();
    ctx->host_threads = hc ? (int)hc : 1;
    *out = ctx.release();
    return 0;
}

void pixo_b200_ctx_destroy(pixo_b200_ctx *ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    delete ctx;
}

const char *pixo_b200_last_error(const pixo_b200_ctx *ctx)
{
    return ctx ? ctx->err.c_str() : g_thread_err.c_str();
}

int pixo_b200_ctx_set_stream(pixo_b200_ctx *ctx, void *cuda_stream)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    cudaStream_t next = cuda_stream ? reinterpret_cast<cudaStream_t>(cuda_stream) : ctx->own_stream;
    if (next == ctx->stream) return 0;
    // Work queued on the old stream still uses the context's scratch, and ctx_sync, ctx_destroy and the
    // scratch's grow-and-free only wait on the current stream: the new stream waits for the old one's
    // work, on the device, so everything queued before the switch is ordered before everything after it.
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    PIXO_CUDA(ctx, cudaEventRecord(ctx->switch_event, ctx->stream));
    PIXO_CUDA(ctx, cudaStreamWaitEvent(next, ctx->switch_event, 0));
    ctx->stream = next;
    return 0;
}

void *pixo_b200_ctx_stream(pixo_b200_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }

int pixo_b200_ctx_sync(pixo_b200_ctx *ctx)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

uint64_t pixo_b200_ctx_launch_count(const pixo_b200_ctx *ctx) { return ctx ? ctx->launches : 0; }

int pixo_b200_ctx_set_host_threads(pixo_b200_ctx *ctx, int n)
{
    if (!ctx || n < 1) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "bad host thread count");
    ctx->host_threads = n;
    return 0;
}

uint64_t pixo_b200_ctx_host_fallbacks(const pixo_b200_ctx *ctx) { return ctx ? ctx->host_fallbacks : 0; }

int pixo_b200_ctx_set_scan_capacity(pixo_b200_ctx *ctx, size_t bytes_per_frame, int gpu_retry)
{
    if (!ctx) return set_error(nullptr, PIXO_B200_ERR_INVALID_ARGUMENT, "ctx is null");
    ctx->scan_cap_override = bytes_per_frame;
    ctx->gpu_retry = gpu_retry != 0;
    return 0;
}

int pixo_b200_dev_alloc(pixo_b200_ctx *ctx, size_t bytes, void **dptr)
{
    if (!ctx || !dptr) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    PIXO_CUDA(ctx, cudaSetDevice(ctx->device));
    PIXO_CUDA(ctx, cudaMalloc(dptr, bytes ? bytes : 1));
    return 0;
}

int pixo_b200_dev_free(pixo_b200_ctx *ctx, void *dptr)
{
    if (!ctx) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    PIXO_CUDA(ctx, cudaFree(dptr));
    return 0;
}

int pixo_b200_host_alloc_pinned(pixo_b200_ctx *ctx, size_t bytes, void **hptr)
{
    if (!ctx || !hptr) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    PIXO_CUDA(ctx, cudaMallocHost(hptr, bytes ? bytes : 1));
    return 0;
}

int pixo_b200_host_free_pinned(pixo_b200_ctx *ctx, void *hptr)
{
    if (!ctx) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    PIXO_CUDA(ctx, cudaFreeHost(hptr));
    return 0;
}

int pixo_b200_upload(pixo_b200_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes)
{
    if (!ctx) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    PIXO_CUDA(ctx, cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

int pixo_b200_download(pixo_b200_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes)
{
    if (!ctx) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "null argument");
    PIXO_CUDA(ctx, cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

}  // extern "C"
