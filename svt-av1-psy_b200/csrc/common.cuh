// common.cuh -- shared host/device plumbing for libsvtav1_b200.so (sm_90a only).
//
// The library mirrors the reference's process-global dispatch model
// (Source/Lib/Codec/aom_dsp_rtcd.c:188, common_dsp_rtcd.c:466): one global context, entry points
// callable concurrently from any encoder worker thread.  Each host-buffer call is one RoundTrip: it
// borrows a "lane" (CUDA stream + pinned staging buffer + device buffer of the same layout) from a
// pool, declares the caller memory it sends and the memory it gets back, launches, and has the
// results written back before it returns -- the reference contract is that outputs are fully
// written on return (SURVEY.md 8b).  There is NO CPU fallback: if the device is missing the entry
// points abort.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <set>
#include <utility>
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
    uint8_t*     d_buf    = nullptr;  // device buffer, same layout as h_buf
    size_t       cap      = 0;
    bool         busy     = false;

    // grow both buffers to at least `bytes`; what they held is not kept
    void reserve(size_t bytes);
};

struct Context {
    int  device      = -1;
    int  sm_count    = 0;
    int  max_smem    = 0;  // opt-in dynamic shared memory per CTA
    bool ready       = false;
    std::mutex          mu;
    std::vector<Lane*>  lanes;
    unsigned long long  launches = 0;  // kernels launched by this library (bench "gpu_launches")
    // device state of one initialisation: svt_b200_shutdown releases or forgets all of it, so that a later svt_b200_init
    // (on the same or another device) meets nothing of the old one
    struct StreamBuf { void* p = nullptr; size_t cap = 0; };
    int                          epoch = 0;      // bumped by every successful svt_b200_init
    std::vector<void*>           scratch;        // every device scratch buffer ever taken: freed at shutdown, never earlier
    std::map<std::pair<const void*, cudaStream_t>, StreamBuf> stream_bufs;  // stream_scratch(): current buffer per (key, stream)
    std::set<const void*>        smem_opted_in;  // allow_dynamic_smem(): kernels whose attribute is set
    std::vector<cudaStream_t>    side_streams;   // ForkJoin handles of all host threads
    std::vector<cudaEvent_t>     side_events;
};

Context& ctx();
void     require_ready();  // aborts loudly when svt_b200_init() has not succeeded
Lane*    lane_acquire();
void     lane_release(Lane* l);
void     count_launch(int n = 1);
// Device scratch of at least `bytes` that belongs to one (key, stream).  `key` is any module-local address (a static tag),
// so calls on different streams never share a buffer, and a call holds no lock across its launches.  A larger request
// takes a new buffer of twice its size; the old one is neither freed nor moved before svt_b200_shutdown(), since a CUDA
// graph captured earlier may still reference it.  A call that needs several arrays carves them at align256() offsets.
void*    stream_scratch(const void* key, cudaStream_t stream, size_t bytes);
static inline size_t align256(size_t bytes) { return (bytes + 255) & ~size_t(255); }
// Lets `kernel` launch with `bytes` of dynamic shared memory (above the 48 KB default): the attribute is set by the first
// call after each initialisation.
void     allow_dynamic_smem(const void* kernel, size_t bytes);
template <typename... A> void allow_dynamic_smem(void (*kernel)(A...), size_t bytes) { allow_dynamic_smem((const void*)kernel, bytes); }
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

// One synchronous host round trip of a T1 (or `_batch_host`) call on a lane.  The call declares regions, launches on
// stream() with dev() pointers, and calls finish().  The first fill() or dev() seals the layout: inputs, then in-outs,
// then outputs, then device-only scratch, each 256-B aligned, with 256 B of slack after the last (kernels may read a
// little past a region); it sizes the lane once and packs the declared inputs.  The first dev() sends inputs and
// in-outs with one copy.  finish() fetches in-outs and outputs with one copy, synchronises, and writes back exactly the
// declared destinations; a call that writes back less than it fetched reads host() after finish() and unpacks by hand.
// Pitches and sizes count elements of T.  A null source leaves a region unpacked; a null destination is not written.
class RoundTrip {
  public:
    template <typename T> struct Buf { int i; };

    RoundTrip() : l_(lane_acquire()) {}
    ~RoundTrip() { lane_release(l_); }
    RoundTrip(const RoundTrip&)            = delete;
    RoundTrip& operator=(const RoundTrip&) = delete;

    // `n_alloc` (> n) sizes a region that must be larger than its data, e.g. for a kernel that reads past it
    template <typename T> Buf<T> in(const T* p, size_t n, size_t n_alloc = 0) {
        return {add(kIn, sizeof(T), n, 1, n_alloc, p, nullptr, n, nullptr, 0)};
    }
    // rows of w elements, packed at pitch w
    template <typename T> Buf<T> in_rows(const T* p, size_t pitch, size_t w, size_t rows) {
        return {add(kIn, sizeof(T), w, rows, 0, p, nullptr, pitch, nullptr, 0)};
    }
    // one row pointer per row (a null row is left unpacked), packed at pitch w
    template <typename T> Buf<T> in_row_list(const T* const* row, size_t w, size_t rows, size_t n_alloc = 0) {
        return {add(kIn, sizeof(T), w, rows, n_alloc, nullptr, reinterpret_cast<const void* const*>(row), 0, nullptr, 0)};
    }
    template <typename T> Buf<T> inout(T* p, size_t n) { return {add(kInOut, sizeof(T), n, 1, 0, p, nullptr, n, p, n)}; }
    template <typename T> Buf<T> out(T* dst, size_t n, size_t n_alloc = 0) {
        return {add(kOut, sizeof(T), n, 1, n_alloc, nullptr, nullptr, 0, dst, n)};
    }
    template <typename T> Buf<T> out_rows(T* dst, size_t pitch, size_t w, size_t rows) {
        return {add(kOut, sizeof(T), w, rows, 0, nullptr, nullptr, 0, dst, pitch)};
    }
    template <typename T> Buf<T> scratch(size_t n) { return {add(kScratch, sizeof(T), n, 1, 0, nullptr, nullptr, 0, nullptr, 0)}; }

    // host view of an input region, to pack by hand what no declaration describes; only before the first dev()
    template <typename T> T* fill(Buf<T> b) {
        if (state_ == kOpen) seal();
        if (state_ != kSealed || slot_[b.i].kind != kIn) misuse("fill() of a region that is not an unsent input");
        return reinterpret_cast<T*>(l_->h_buf + slot_[b.i].off);
    }
    template <typename T> T* dev(Buf<T> b) {
        if (state_ != kSent) send();
        return reinterpret_cast<T*>(l_->d_buf + slot_[b.i].off);
    }
    cudaStream_t stream() const { return l_->stream; }
    void         finish();
    template <typename T> T* host(Buf<T> b) {
        if (state_ != kDone) misuse("host() before finish()");
        return reinterpret_cast<T*>(l_->h_buf + slot_[b.i].off);
    }

  private:
    enum Kind : uint8_t { kIn, kInOut, kOut, kScratch };
    enum State : uint8_t { kOpen, kSealed, kSent, kDone };
    struct Slot {
        Kind               kind;
        size_t             bytes, off;       // the region
        size_t             row_bytes, rows;  // what is packed into it / written back from it, at pitch row_bytes
        const uint8_t*     src;              // packed from rows at src_pitch ...
        const void* const* src_row;          // ... or from one pointer per row
        size_t             src_pitch;
        uint8_t*           dst;              // written back to rows at dst_pitch
        size_t             dst_pitch;
    };
    static constexpr int kSlots = 8;

    int  add(Kind kind, size_t elem, size_t w, size_t rows, size_t n_alloc, const void* src, const void* const* src_row,
             size_t src_pitch, void* dst, size_t dst_pitch);
    void seal();
    void send();
    [[noreturn]] static void misuse(const char* what);

    Lane*  l_;
    Slot   slot_[kSlots];
    int    n_     = 0;
    State  state_ = kOpen;
    size_t h2d_bytes_ = 0, d2h_off_ = 0, d2h_bytes_ = 0;
};

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
