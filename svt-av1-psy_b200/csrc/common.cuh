// common.cuh -- shared host/device plumbing for libsvtav1_b200.so (sm_90a only).
//
// The library mirrors the reference's process-global dispatch model
// (Source/Lib/Codec/aom_dsp_rtcd.c:188, common_dsp_rtcd.c:466): one global context, entry points
// callable concurrently from any encoder worker thread.  Each host-buffer call borrows a "lane"
// (CUDA stream + pinned staging buffer + device scratch) from a pool, stages the caller-owned host
// memory, launches, and copies results back before returning -- the reference contract is that
// outputs are fully written on return (SURVEY.md 8b).  There is NO CPU fallback: if the device is
// missing the entry points abort.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#define B200_CUDA_CHECK(expr)                                                                    \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess) {                                                                 \
            fprintf(stderr, "[svt_b200] FATAL %s:%d: %s -> %s\n", __FILE__, __LINE__, #expr,     \
                    cudaGetErrorString(_e));                                                     \
            abort();                                                                             \
        }                                                                                        \
    } while (0)

namespace b200 {

struct Lane {
    cudaStream_t stream   = nullptr;
    uint8_t*     h_buf    = nullptr;  // pinned host staging
    uint8_t*     d_buf    = nullptr;  // device scratch, same layout as h_buf
    size_t       cap      = 0;
    size_t       used     = 0;
    bool         busy     = false;

    void reserve(size_t bytes);
    // bump-allocate `bytes` (256-B aligned) in both buffers; returns the offset
    size_t alloc(size_t bytes) {
        size_t off = (used + 255) & ~size_t(255);
        reserve(off + bytes + 256);
        used = off + bytes;
        return off;
    }
    template <typename T> T* h(size_t off) { return reinterpret_cast<T*>(h_buf + off); }
    template <typename T> T* d(size_t off) { return reinterpret_cast<T*>(d_buf + off); }
    void h2d(size_t off, size_t bytes) {
        if (bytes) B200_CUDA_CHECK(cudaMemcpyAsync(d_buf + off, h_buf + off, bytes, cudaMemcpyHostToDevice, stream));
    }
    void d2h(size_t off, size_t bytes) {
        if (bytes) B200_CUDA_CHECK(cudaMemcpyAsync(h_buf + off, d_buf + off, bytes, cudaMemcpyDeviceToHost, stream));
    }
    void sync() { B200_CUDA_CHECK(cudaStreamSynchronize(stream)); }
};

struct Context {
    int  device      = -1;
    int  sm_count    = 0;
    int  max_smem    = 0;  // opt-in dynamic shared memory per CTA
    bool ready       = false;
    std::mutex          mu;
    std::vector<Lane*>  lanes;
    unsigned long long  launches = 0;  // kernels launched by this library (bench "gpu_launches")
    // lifetime of module state (svt_b200_shutdown -> svt_b200_init on another device must not meet anything of the old one)
    int                          epoch = 0;      // bumped by every successful svt_b200_init
    std::vector<void*>           scratch;        // every device scratch buffer of every module: freed at shutdown, never earlier
    std::vector<void (*)()>      resets;         // per-module "forget your cached pointers" hooks
    std::vector<cudaStream_t>    side_streams;   // ForkJoin handles of all host threads
    std::vector<cudaEvent_t>     side_events;
};

Context& ctx();
void     require_ready();  // aborts loudly when svt_b200_init() has not succeeded
Lane*    lane_acquire();
void     lane_release(Lane* l);
void     count_launch(int n = 1);
// Device scratch owned by the library.  A module that outgrows a buffer takes a new one and leaves the old one alone:
// a CUDA graph captured earlier may still reference it.  Everything is released by svt_b200_shutdown().
void*    scratch_alloc(size_t bytes);
void     register_reset(void (*fn)());  // fn drops the module's cached scratch pointers / capacities (called at shutdown)
int      epoch();                       // changes with every (re-)initialisation: per-function attributes are re-applied
struct ResetHook { explicit ResetHook(void (*fn)()) { register_reset(fn); } };
void     txfm_tables_init();  // txfm.cu: uploads the transform constant tables

// Side streams for calls whose launches are independent of each other: fork_streams() makes the side
// streams wait for everything already enqueued on `user`, join_streams() makes `user` wait for them.
// One set per host thread (events are re-recorded call after call; a wait keeps the record it saw).
struct ForkJoin {
    static constexpr int kSide = 3;
    cudaStream_t side[kSide];
    cudaEvent_t  forked, done[kSide];
    int          epoch = -1;  // the initialisation these handles belong to
};
ForkJoin& fork_streams(cudaStream_t user);
void      join_streams(ForkJoin& fj, cudaStream_t user);

struct LaneGuard {
    Lane* l;
    LaneGuard() : l(lane_acquire()) {}
    ~LaneGuard() { lane_release(l); }
    Lane* operator->() { return l; }
};

// copy a strided 2-D host region into a packed staging area
static inline void copy2d(uint8_t* dst, size_t dpitch, const uint8_t* src, size_t spitch, size_t wbytes, size_t rows) {
    for (size_t r = 0; r < rows; r++) memcpy(dst + r * dpitch, src + r * spitch, wbytes);
}

static inline int grid_for(long long work_ctas, int ctas_per_sm = 8) {
    long long cap = (long long)ctx().sm_count * ctas_per_sm;
    if (work_ctas < 1) work_ctas = 1;
    return (int)(work_ctas < cap ? work_ctas : cap);
}

}  // namespace b200

#define B200_LAUNCH_CHECK()                        \
    do {                                           \
        B200_CUDA_CHECK(cudaGetLastError());       \
        b200::count_launch();                      \
    } while (0)
