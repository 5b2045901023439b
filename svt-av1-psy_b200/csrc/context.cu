// context.cu -- device bring-up, lane pool.  See include/svt_b200.h.
#include "common.cuh"
#include "../../include/svt_b200.h"

namespace b200 {

static Context g_ctx;
Context& ctx() { return g_ctx; }

// A round trip sizes its lane once, before it packs anything, and every round trip synchronises before it releases the
// lane: the old buffers hold nothing and nothing is in flight on them.
void Lane::reserve(size_t bytes) {
    if (bytes <= cap) return;
    size_t ncap = cap ? cap : (size_t(4) << 20);
    while (ncap < bytes) ncap *= 2;
    if (h_buf) {
        B200_CUDA_CHECK(cudaFreeHost(h_buf));
        B200_CUDA_CHECK(cudaFree(d_buf));
    }
    B200_CUDA_CHECK(cudaHostAlloc(&h_buf, ncap, cudaHostAllocDefault));
    B200_CUDA_CHECK(cudaMalloc(&d_buf, ncap));
    cap = ncap;
}

static void copy2d(uint8_t* dst, size_t dpitch, const uint8_t* src, size_t spitch, size_t wbytes, size_t rows) {
    for (size_t r = 0; r < rows; r++) memcpy(dst + r * dpitch, src + r * spitch, wbytes);
}

void RoundTrip::misuse(const char* what) {
    fprintf(stderr, "[svt_b200] FATAL: round trip: %s\n", what);
    abort();
}

int RoundTrip::add(Kind kind, size_t elem, size_t w, size_t rows, size_t n_alloc, const void* src, const void* const* src_row,
                   size_t src_pitch, void* dst, size_t dst_pitch) {
    if (state_ != kOpen) misuse("region declared after the layout was sealed");
    if (n_ == kSlots) misuse("more regions than the slot table holds");
    Slot& s     = slot_[n_];
    s.kind      = kind;
    s.row_bytes = w * elem;
    s.rows      = rows;
    s.bytes     = n_alloc > w * rows ? n_alloc * elem : s.row_bytes * rows;
    s.src       = static_cast<const uint8_t*>(src);
    s.src_row   = src_row;
    s.src_pitch = src_pitch * elem;
    s.dst       = static_cast<uint8_t*>(dst);
    s.dst_pitch = dst_pitch * elem;
    return n_++;
}

void RoundTrip::seal() {
    size_t end = 0, d2h_off = ~size_t(0);
    for (int k = kIn; k <= kScratch; k++) {
        for (int i = 0; i < n_; i++) {
            Slot& s = slot_[i];
            if (s.kind != k) continue;
            s.off = align256(end);
            end   = s.off + s.bytes;
            if ((k == kInOut || k == kOut) && d2h_off == ~size_t(0)) d2h_off = s.off;
        }
        if (k == kInOut) h2d_bytes_ = end;
        if (k == kOut && d2h_off != ~size_t(0)) {
            d2h_off_   = d2h_off;
            d2h_bytes_ = end - d2h_off;
        }
    }
    l_->reserve(end + 256);
    for (int i = 0; i < n_; i++) {
        const Slot& s = slot_[i];
        uint8_t*    h = l_->h_buf + s.off;
        if (s.src_row) {
            for (size_t r = 0; r < s.rows; r++)
                if (s.src_row[r]) memcpy(h + r * s.row_bytes, s.src_row[r], s.row_bytes);
        } else if (s.src) {
            copy2d(h, s.row_bytes, s.src, s.src_pitch, s.row_bytes, s.rows);
        }
    }
    state_ = kSealed;
}

void RoundTrip::send() {
    if (state_ == kDone) misuse("dev() after finish()");
    if (state_ == kOpen) seal();
    if (h2d_bytes_) B200_CUDA_CHECK(cudaMemcpyAsync(l_->d_buf, l_->h_buf, h2d_bytes_, cudaMemcpyHostToDevice, l_->stream));
    state_ = kSent;
}

void RoundTrip::finish() {
    if (state_ != kSent) send();
    if (d2h_bytes_)
        B200_CUDA_CHECK(cudaMemcpyAsync(l_->h_buf + d2h_off_, l_->d_buf + d2h_off_, d2h_bytes_, cudaMemcpyDeviceToHost, l_->stream));
    B200_CUDA_CHECK(cudaStreamSynchronize(l_->stream));
    for (int i = 0; i < n_; i++) {
        const Slot& s = slot_[i];
        if (s.dst) copy2d(s.dst, s.dst_pitch, l_->h_buf + s.off, s.row_bytes, s.row_bytes, s.rows);
    }
    state_ = kDone;
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

void* stream_scratch(const void* key, cudaStream_t stream, size_t bytes) {
    std::lock_guard<std::mutex> lk(g_ctx.mu);
    Context::StreamBuf& b = g_ctx.stream_bufs[{key, stream}];
    if (bytes > b.cap) {
        b.cap = bytes * 2;
        B200_CUDA_CHECK(cudaMalloc(&b.p, b.cap));
        g_ctx.scratch.push_back(b.p);
    }
    return b.p;
}

void allow_dynamic_smem(const void* kernel, size_t bytes) {
    std::lock_guard<std::mutex> lk(g_ctx.mu);
    if (g_ctx.smem_opted_in.insert(kernel).second)
        B200_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
}

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
    for (void* p : c.scratch) cudaFree(p);  // nothing was freed before: captured graphs may have referenced any of it
    c.scratch.clear();
    c.stream_bufs.clear();
    c.smem_opted_in.clear();
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
