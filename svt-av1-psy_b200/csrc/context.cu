// context.cu -- device bring-up, lane pool.  See include/svt_b200.h.
#include "common.cuh"
#include "../../include/svt_b200.h"

namespace b200 {

static Context g_ctx;
Context& ctx() { return g_ctx; }

void Lane::reserve(size_t bytes) {
    if (bytes <= cap) return;
    size_t ncap = cap ? cap : (size_t(4) << 20);
    while (ncap < bytes) ncap *= 2;
    uint8_t* nh = nullptr;
    uint8_t* nd = nullptr;
    B200_CUDA_CHECK(cudaHostAlloc(&nh, ncap, cudaHostAllocDefault));
    B200_CUDA_CHECK(cudaMalloc(&nd, ncap));
    if (h_buf) {
        // growing in the middle of a call: preserve what was staged so far
        B200_CUDA_CHECK(cudaStreamSynchronize(stream));
        memcpy(nh, h_buf, used);
        B200_CUDA_CHECK(cudaMemcpy(nd, d_buf, used, cudaMemcpyDeviceToDevice));
        B200_CUDA_CHECK(cudaFreeHost(h_buf));
        B200_CUDA_CHECK(cudaFree(d_buf));
    }
    h_buf = nh;
    d_buf = nd;
    cap   = ncap;
}

void require_ready() {
    if (!g_ctx.ready) {
        fprintf(stderr,
                "[svt_b200] FATAL: entry point called before a successful svt_b200_init(); this "
                "library has no CPU fallback.\n");
        abort();
    }
    // Encoder worker threads (and host frameworks sharing the process) may have another CUDA
    // context / device current on this thread: always re-bind the library's device first.
    B200_CUDA_CHECK(cudaSetDevice(g_ctx.device));
}

Lane* lane_acquire() {
    require_ready();
    std::lock_guard<std::mutex> lk(g_ctx.mu);
    for (Lane* l : g_ctx.lanes)
        if (!l->busy) {
            l->busy = true;
            l->used = 0;
            B200_CUDA_CHECK(cudaSetDevice(g_ctx.device));
            return l;
        }
    B200_CUDA_CHECK(cudaSetDevice(g_ctx.device));
    Lane* l = new Lane();
    B200_CUDA_CHECK(cudaStreamCreateWithFlags(&l->stream, cudaStreamNonBlocking));
    l->busy = true;
    g_ctx.lanes.push_back(l);
    return l;
}

void lane_release(Lane* l) {
    std::lock_guard<std::mutex> lk(g_ctx.mu);
    l->busy = false;
}

void* scratch_alloc(size_t bytes) {
    void* p = nullptr;
    B200_CUDA_CHECK(cudaMalloc(&p, bytes ? bytes : 1));
    std::lock_guard<std::mutex> lk(g_ctx.mu);
    g_ctx.scratch.push_back(p);
    return p;
}
// the hooks register from static initialisers of other translation units: the list must not depend on the construction
// order of namespace-scope objects, hence function-local statics
static std::vector<void (*)()>& reset_list() { static std::vector<void (*)()> v; return v; }
static std::mutex& reset_mu() { static std::mutex m; return m; }
void register_reset(void (*fn)()) {
    std::lock_guard<std::mutex> lk(reset_mu());
    reset_list().push_back(fn);
}
int epoch() { return g_ctx.epoch; }

void count_launch(int n) { __atomic_fetch_add(&g_ctx.launches, (unsigned long long)n, __ATOMIC_RELAXED); }

}  // namespace b200

using namespace b200;

extern "C" int svt_b200_init(int device) {
    Context& c = ctx();
    std::lock_guard<std::mutex> lk(c.mu);
    if (c.ready) return c.device == device || device < 0 ? SVT_B200_OK : SVT_B200_ERR_ALREADY_INIT;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) return SVT_B200_ERR_NO_DEVICE;
    if (device < 0) device = 0;
    if (device >= n) return SVT_B200_ERR_NO_DEVICE;
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, device) != cudaSuccess) return SVT_B200_ERR_NO_DEVICE;
    if (p.major != 9) {
        fprintf(stderr, "[svt_b200] device %d is sm_%d%d; this library is built for sm_90a only\n", device, p.major,
                p.minor);
        return SVT_B200_ERR_BAD_ARCH;
    }
    if (cudaSetDevice(device) != cudaSuccess) return SVT_B200_ERR_NO_DEVICE;
    c.device   = device;
    c.sm_count = p.multiProcessorCount;
    c.max_smem = (int)p.sharedMemPerBlockOptin;
    txfm_tables_init();
    c.epoch++;
    c.ready    = true;
    return SVT_B200_OK;
}

extern "C" void svt_b200_shutdown(void) {
    Context& c = ctx();
    std::lock_guard<std::mutex> lk(c.mu);
    if (!c.ready) return;
    cudaSetDevice(c.device);
    for (Lane* l : c.lanes) {
        cudaStreamSynchronize(l->stream);
        if (l->h_buf) cudaFreeHost(l->h_buf);
        if (l->d_buf) cudaFree(l->d_buf);
        cudaStreamDestroy(l->stream);
        delete l;
    }
    c.lanes.clear();
    cudaDeviceSynchronize();
    {
        std::lock_guard<std::mutex> rl(reset_mu());
        for (void (*fn)() : reset_list()) fn();   // modules forget their cached scratch / per-stream state ...
    }
    if (false) for (void (*fn)() : c.resets) fn();           // modules forget their cached scratch / per-stream state ...
    for (void* p : c.scratch) cudaFree(p);        // ... and the scratch itself goes (nothing was freed before: captured graphs)
    c.scratch.clear();
    for (cudaStream_t s : c.side_streams) cudaStreamDestroy(s);
    for (cudaEvent_t e : c.side_events) cudaEventDestroy(e);
    c.side_streams.clear();
    c.side_events.clear();
    c.ready = false;
}

// plain asynchronous copies on a caller stream (the host-buffer side of the T2 calls: pinned host <-> device, device <-> device)
extern "C" int svt_b200_copy_async(void* dst, const void* src, size_t bytes, int kind, void* stream) {
    if (!dst || !src || kind < 0 || kind > 2) return SVT_B200_ERR_BAD_ARG;
    const cudaMemcpyKind k = kind == 0 ? cudaMemcpyHostToDevice : (kind == 1 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice);
    if (bytes) B200_CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, k, (cudaStream_t)stream));
    return SVT_B200_OK;
}
extern "C" int svt_b200_copy2d_async(void* dst, size_t dst_pitch, const void* src, size_t src_pitch, size_t width_bytes, size_t rows, int kind,
                                     void* stream) {
    if (!dst || !src || kind < 0 || kind > 2) return SVT_B200_ERR_BAD_ARG;
    const cudaMemcpyKind k = kind == 0 ? cudaMemcpyHostToDevice : (kind == 1 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice);
    if (width_bytes && rows) B200_CUDA_CHECK(cudaMemcpy2DAsync(dst, dst_pitch, src, src_pitch, width_bytes, rows, k, (cudaStream_t)stream));
    return SVT_B200_OK;
}

extern "C" int svt_b200_sm_count(void) { return ctx().ready ? ctx().sm_count : 0; }
extern "C" unsigned long long svt_b200_launch_count(void) { return ctx().launches; }
extern "C" const char* svt_b200_version(void) { return "svt_b200 0.1 (sm_90a)"; }

namespace b200 {

ForkJoin& fork_streams(cudaStream_t user) {
    static thread_local ForkJoin fj;
    if (fj.epoch != g_ctx.epoch) {  // first use by this host thread, or the library was shut down and re-initialised since
        for (int i = 0; i < ForkJoin::kSide; i++) {
            B200_CUDA_CHECK(cudaStreamCreateWithFlags(&fj.side[i], cudaStreamNonBlocking));
            B200_CUDA_CHECK(cudaEventCreateWithFlags(&fj.done[i], cudaEventDisableTiming));
        }
        B200_CUDA_CHECK(cudaEventCreateWithFlags(&fj.forked, cudaEventDisableTiming));
        {
            std::lock_guard<std::mutex> lk(g_ctx.mu);
            for (int i = 0; i < ForkJoin::kSide; i++) {
                g_ctx.side_streams.push_back(fj.side[i]);
                g_ctx.side_events.push_back(fj.done[i]);
            }
            g_ctx.side_events.push_back(fj.forked);
        }
        fj.epoch = g_ctx.epoch;
    }
    B200_CUDA_CHECK(cudaEventRecord(fj.forked, user));
    for (int i = 0; i < ForkJoin::kSide; i++) B200_CUDA_CHECK(cudaStreamWaitEvent(fj.side[i], fj.forked, 0));
    return fj;
}

void join_streams(ForkJoin& fj, cudaStream_t user) {
    for (int i = 0; i < ForkJoin::kSide; i++) {
        B200_CUDA_CHECK(cudaEventRecord(fj.done[i], fj.side[i]));
        B200_CUDA_CHECK(cudaStreamWaitEvent(user, fj.done[i], 0));
    }
}

}  // namespace b200
