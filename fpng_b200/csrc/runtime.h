// fpng_b200/csrc/runtime.h -- host runtime state shared by host_api.cu and decode_api.cu.
#pragma once
#include "../../include/fpng_b200.h"
#include "common.cuh"
#include <mutex>
#include <new>
#include <vector>

namespace fpngb {

struct Buffer {
    void* p = nullptr; size_t cap = 0; bool pinned = false;
    int reserve(size_t n)
    {
        if (n <= cap) return 0;
        if (p) { if (pinned) cudaFreeHost(p); else cudaFree(p); p = nullptr; cap = 0; }
        n = (n + (1u << 20)) & ~((size_t)(1u << 20) - 1);
        FPNGB_CUDA_OK(pinned ? cudaMallocHost(&p, n) : cudaMalloc(&p, n));
        cap = n;
        return 0;
    }
};

// One pinned buffer of the staging ring for host-built tables that a call uploads (descriptor tables, offsets).  The caller
// records ev on the stream after the copies that read buf.
struct StageSlot { Buffer buf; cudaEvent_t ev = nullptr; };

struct Context {
    int device = -1;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_in = nullptr, copy_out = nullptr;   // H2D / D2H streams of the pipelined host batch path
    cudaStream_t side = nullptr;                 // CRC kernels of one chunk run here underneath the scan/pack kernels of the next
    cudaEvent_t side_ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    const uint32_t* crc_f128b = nullptr;        // device tables of the in-kernel CRC (crc_stream_kernel.cu)
    const uint32_t* crc_lane_mul = nullptr;
    CodeBook* d_static_books = nullptr;          // [0] RGB, [1] RGBA
    CodeBook h_static_books[2];
    Buffer ws;                                    // kernel workspace (row tables, image state, histograms, books)
    Buffer conv;                                  // uint8 images the *_typed encode calls convert their input into (used under ws_acquire)
    Buffer red;                                   // FPNGB_ENCODE_REDUCE: per-image analysis state, colour sets and results (under ws_acquire)
    Buffer dev_in, dev_out;                       // staging for the *_host entry points
    Buffer pin_small;                             // pinned scratch for sizes / status words
    std::mutex mu;                                // the *_host entry points and the workspace are serialised
    bool ready = false;
    // The workspaces are shared by consecutive batch calls: work enqueued on a different stream than the previous call
    // first waits (on the device) for that call's kernels.
    cudaEvent_t ws_done = nullptr;
    cudaStream_t ws_stream = nullptr;
    bool ws_busy = false;
    int ws_acquire(cudaStream_t s)
    {
        if (!ws_done) FPNGB_CUDA_OK(cudaEventCreateWithFlags(&ws_done, cudaEventDisableTiming));
        if (ws_busy && ws_stream != s) FPNGB_CUDA_OK(cudaStreamWaitEvent(s, ws_done, 0));
        return 0;
    }
    int ws_release(cudaStream_t s)
    {
        FPNGB_CUDA_OK(cudaEventRecord(ws_done, s));
        ws_stream = s; ws_busy = true;
        return 0;
    }
    // A staging slot of at least `bytes`: one whose last copy has completed (cudaEventQuery), else a new one, so that a call never
    // waits on the host for an earlier call's upload.  Slots live as long as the process.
    std::vector<StageSlot*> stage;
    int stage_slot(size_t bytes, StageSlot** out)
    {
        StageSlot* sl = nullptr;
        for (StageSlot* x : stage) if (x->buf.cap >= bytes && cudaEventQuery(x->ev) == cudaSuccess) { sl = x; break; }
        if (!sl) {
            sl = new (std::nothrow) StageSlot();
            if (!sl) return FPNGB_ERR_INTERNAL;
            sl->buf.pinned = true;
            FPNGB_CUDA_OK(cudaEventCreateWithFlags(&sl->ev, cudaEventDisableTiming));
            stage.push_back(sl);
        }
        const int rc = sl->buf.reserve(bytes);
        if (rc) return rc;
        *out = sl;
        return 0;
    }
};


// a fixed set of timing-less events that is destroyed on every exit path of the pipelined host entry points
template <int N>
struct EventSet {
    cudaEvent_t ev[N];
    bool ok = true;
    EventSet() { for (int i = 0; i < N; i++) { ev[i] = nullptr; if (cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming) != cudaSuccess) ok = false; } }
    ~EventSet() { for (int i = 0; i < N; i++) if (ev[i]) cudaEventDestroy(ev[i]); }
    EventSet(const EventSet&) = delete;
    EventSet& operator=(const EventSet&) = delete;
};

Context& context();
void count_launch(uint64_t n);
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace fpngb
