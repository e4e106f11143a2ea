// Device / stream plumbing for the hot paths.
//
// Plays the role of the reference's util/gpu_t.cuh (gpu_t, stream_t, select_gpu, CUDA_OK;
// util/gpu_t.cuh:20-267, util/exception.cuh:12-21) with the same public names, redesigned
// around stream-ordered allocation: one gpu_t per visible device, every scratch buffer comes
// from the device's cudaMemPool (no cudaMalloc on the hot path once the pool is warm), and
// work can be enqueued on a caller-supplied stream (PyTorch's current stream in bench.py).
#pragma once
#include <cuda_runtime.h>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <algorithm>
#include <stdexcept>
#include <string>
#include <vector>
#include "../../../include/sppark_b200.h"

class cuda_error : public std::runtime_error {
    int _code;
public:
    cuda_error(int code, const std::string& what) : std::runtime_error(what), _code(code) {}
    int code() const { return _code; }
};

#define CUDA_OK(expr) do {                                                          \
    cudaError_t _e = (expr);                                                        \
    if (_e != cudaSuccess) {                                                        \
        (void)cudaGetLastError();                                                   \
        throw cuda_error(-(int)_e, std::string(cudaGetErrorString(_e)) + " @" +     \
                         __FILE__ + ":" + std::to_string(__LINE__));                \
    }                                                                               \
} while (0)

inline RustError rust_ok() { return RustError{0, nullptr}; }
inline RustError rust_err(int code, const std::string& msg)
{   return RustError{code, msg.empty() ? nullptr : strdup(msg.c_str())};   }

// fn() for a C entry point: what it throws becomes the returned error instead of leaving the library
template<class Fn> RustError guarded(Fn&& fn)
{
    try {
        return fn();
    } catch (const cuda_error& e) {
        return rust_err(e.code(), e.what());
    } catch (const std::exception& e) {
        return rust_err(-1, e.what());
    }
}

// raises kernel K's dynamic shared-memory limit to `bytes` once per device (function attributes
// are per device context); static, as every translation unit has its own copy of a kernel
template<auto K> static void smem_opt_in(int dev, int bytes)
{
    static bool done[64];
    if (!done[dev & 63]) {
        CUDA_OK(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        done[dev & 63] = true;
    }
}

extern std::atomic<uint64_t> g_launch_count;      // defined in api.cu

// Optional phase timing (bench.py's roofline leg): when enabled, the drivers drop CUDA events
// on their own stream at phase boundaries of the LAST call; sppark_b200_profile_read() turns
// them into milliseconds once the caller has synchronised.  Off by default (no events).
struct phase_profile_t {
    static constexpr int MAX = 16;
    bool enabled = false;
    int n = 0;
    cudaEvent_t ev[MAX] = {};
    const char* name[MAX] = {};
    void mark(const char* what, cudaStream_t s)
    {
        if (!enabled || n >= MAX) return;
        if (!ev[n]) cudaEventCreate(&ev[n]);
        cudaEventRecord(ev[n], s);
        name[n++] = what;
    }
    void reset() { n = 0; }
};
extern phase_profile_t g_profile;
#define COUNT_LAUNCH() (g_launch_count.fetch_add(1, std::memory_order_relaxed))

class stream_t {
    cudaStream_t s;
    bool owned;
public:
    explicit stream_t(cudaStream_t borrowed) : s(borrowed), owned(false) {}
    stream_t() : owned(true) { CUDA_OK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)); }
    ~stream_t() { if (owned) cudaStreamDestroy(s); }
    stream_t(const stream_t&) = delete;
    operator cudaStream_t() const { return s; }

    void* Dmalloc(size_t bytes) const
    {   void* p; CUDA_OK(cudaMallocAsync(&p, bytes ? bytes : 1, s)); return p;   }
    void Dfree(void* p) const { if (p) (void)cudaFreeAsync(p, s); }
    void HtoD(void* dst, const void* src, size_t bytes) const
    {   CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s));   }
    void DtoH(void* dst, const void* src, size_t bytes) const
    {   CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s));   }
    // strided host rows -> packed device rows (reference: stream_t::HtoD with pitch, util/gpu_t.cuh:84-93)
    void HtoD2D(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t rows) const
    {   CUDA_OK(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, rows, cudaMemcpyHostToDevice, s));   }
    void sync() const { CUDA_OK(cudaStreamSynchronize(s)); }
};

// On a failure, waits for the work of one or two streams while the buffers it uses are still alive
// (their stream-ordered frees run during unwinding); disarmed once the call has synchronised.
class drain_t {
    const stream_t &a, &b;
public:
    bool armed = true;
    explicit drain_t(const stream_t& s) : a(s), b(s) {}
    drain_t(const stream_t& s, const stream_t& t) : a(s), b(t) {}
    drain_t(const drain_t&) = delete;
    ~drain_t()
    {
        if (!armed) return;
        (void)cudaStreamSynchronize(a);
        if (&b != &a) (void)cudaStreamSynchronize(b);
    }
};

// cudaEvent_t with a lifetime (no timing): destroyed on every exit path
class event_t {
    cudaEvent_t e;
public:
    event_t() { CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); }
    ~event_t() { (void)cudaEventDestroy(e); }
    event_t(const event_t&) = delete;
    operator cudaEvent_t() const { return e; }
    void record(cudaStream_t s) const { CUDA_OK(cudaEventRecord(e, s)); }
    void wait(cudaStream_t s) const { CUDA_OK(cudaStreamWaitEvent(s, e, 0)); }
};

// ---- pageable host memory -> device, at pinned-memory speed ---------------------------------
// cudaMemcpyAsync from pageable memory is staged by the driver through a small bounce buffer on
// the calling thread (~10 GB/s).  The reference's callers (Rust Vec, Go slices) hand over
// pageable memory, so the host-pointer entry points stage it themselves: worker threads copy
// 32 MiB chunks into a ring of pinned buffers while earlier chunks are in flight on the copy
// engine.  Reference counterpart: the host thread pool of gpu_t (util/gpu_t.cuh:176-186,
// util/thread_pool_t.hpp), used there for the post-processing of results.
class stager_t {
    static constexpr size_t CHUNK = (size_t)32 << 20;
    static constexpr int NBUF = 4, NTHREADS = 8;
    uint8_t* buf[NBUF] = {};
    cudaEvent_t ev[NBUF] = {};
    int next = 0;
    std::vector<std::thread> workers;
    std::mutex mtx;
    std::condition_variable cv_work, cv_done;
    struct job_t { uint8_t* dst; const uint8_t* src; size_t len; };
    std::vector<job_t> jobs;
    size_t pending = 0;
    bool quit = false;

    void worker()
    {
        for (;;) {
            job_t j;
            {
                std::unique_lock<std::mutex> lk(mtx);
                cv_work.wait(lk, [&] { return quit || !jobs.empty(); });
                if (quit && jobs.empty()) return;
                j = jobs.back();
                jobs.pop_back();
            }
            memcpy(j.dst, j.src, j.len);
            {
                std::lock_guard<std::mutex> lk(mtx);
                if (--pending == 0) cv_done.notify_all();
            }
        }
    }
    void parallel_copy(uint8_t* dst, const uint8_t* src, size_t len)
    {
        const size_t piece = (len + NTHREADS - 1) / NTHREADS;
        {
            std::lock_guard<std::mutex> lk(mtx);
            for (size_t off = 0; off < len; off += piece) {
                jobs.push_back({dst + off, src + off, std::min(piece, len - off)});
                pending++;
            }
        }
        cv_work.notify_all();
        std::unique_lock<std::mutex> lk(mtx);
        cv_done.wait(lk, [&] { return pending == 0; });
    }

public:
    stager_t()
    {
        for (int i = 0; i < NBUF; i++) {
            CUDA_OK(cudaHostAlloc((void**)&buf[i], CHUNK, cudaHostAllocDefault));
            CUDA_OK(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
        }
        for (int i = 0; i < NTHREADS; i++) workers.emplace_back([this] { worker(); });
    }
    ~stager_t()
    {
        {
            std::lock_guard<std::mutex> lk(mtx);
            quit = true;
        }
        cv_work.notify_all();
        for (auto& t : workers) t.join();
        for (int i = 0; i < NBUF; i++) { cudaFreeHost(buf[i]); cudaEventDestroy(ev[i]); }
    }
    static bool is_pageable(const void* p)
    {
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { (void)cudaGetLastError(); return true; }
        return a.type == cudaMemoryTypeUnregistered;
    }
    // dst (device) <- src (pageable host), enqueued on `s`; returns once the LAST chunk has been
    // handed to the copy engine (the source may not be modified until the stream is synchronised)
    void HtoD(cudaStream_t s, void* dst, const void* src, size_t bytes)
    {
        for (size_t off = 0; off < bytes; off += CHUNK) {
            const int b = next++ % NBUF;
            const size_t len = std::min(CHUNK, bytes - off);
            CUDA_OK(cudaEventSynchronize(ev[b]));            // this ring slot has left the host
            parallel_copy(buf[b], (const uint8_t*)src + off, len);
            CUDA_OK(cudaMemcpyAsync((uint8_t*)dst + off, buf[b], len, cudaMemcpyHostToDevice, s));
            CUDA_OK(cudaEventRecord(ev[b], s));
        }
    }
    // dst (pageable host) <- src (device): chunks land in the pinned ring and are copied out by
    // the workers while the next chunk is on the wire.  Returns when dst is complete.
    void DtoH(cudaStream_t s, void* dst, const void* src, size_t bytes)
    {
        size_t issued = 0, drained = 0;
        int slot_of[NBUF];
        size_t off_of[NBUF], len_of[NBUF];
        int head = 0, tail = 0, inflight = 0;
        while (drained < bytes) {
            while (inflight < NBUF && issued < bytes) {
                const int b = next++ % NBUF;
                const size_t len = std::min(CHUNK, bytes - issued);
                CUDA_OK(cudaEventSynchronize(ev[b]));
                CUDA_OK(cudaMemcpyAsync(buf[b], (const uint8_t*)src + issued, len, cudaMemcpyDeviceToHost, s));
                CUDA_OK(cudaEventRecord(ev[b], s));
                slot_of[head] = b; off_of[head] = issued; len_of[head] = len;
                head = (head + 1) % NBUF;
                issued += len;
                inflight++;
            }
            const int b = slot_of[tail];
            CUDA_OK(cudaEventSynchronize(ev[b]));
            parallel_copy((uint8_t*)dst + off_of[tail], buf[b], len_of[tail]);
            drained += len_of[tail];
            tail = (tail + 1) % NBUF;
            inflight--;
        }
    }
};

// stream-ordered scratch buffer
template<typename T> class dev_ptr_t {
    T* p;
    const stream_t& st;
public:
    dev_ptr_t(size_t n, const stream_t& s) : p((T*)s.Dmalloc(n * sizeof(T))), st(s) {}
    ~dev_ptr_t() { st.Dfree(p); }
    dev_ptr_t(const dev_ptr_t&) = delete;
    operator T*() const { return p; }
    T* get() const { return p; }
};

class gpu_t {
    int gpu_id, cuda_id;
    cudaDeviceProp prop;
    std::unique_ptr<stream_t> streams[3];
public:
    std::mutex cache_mtx;                                   // guards per-device table caches
    std::map<uint64_t, void*> cache;
    mutable std::mutex stage_mtx;                           // one pageable upload at a time
    mutable std::unique_ptr<stager_t> stage;
    stager_t& stager() const
    {
        if (!stage) stage.reset(new stager_t());
        return *stage;
    }

    gpu_t(int id, int cid) : gpu_id(id), cuda_id(cid)
    {
        CUDA_OK(cudaSetDevice(cid));
        CUDA_OK(cudaGetDeviceProperties(&prop, cid));
        for (auto& s : streams) s.reset(new stream_t());
        cudaMemPool_t pool;
        CUDA_OK(cudaDeviceGetDefaultMemPool(&pool, cid));
        uint64_t keep = ~0ull;                              // keep freed scratch in the pool
        CUDA_OK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
        // the point-arithmetic helpers that are deliberately NOT inlined (xyzz add/dbl, the
        // outlined Montgomery ladder) keep their operands on the local-memory stack
        CUDA_OK(cudaDeviceSetLimit(cudaLimitStackSize, 4096));
    }
    int id() const { return gpu_id; }
    int cid() const { return cuda_id; }
    int sm_count() const { return prop.multiProcessorCount; }
    const cudaDeviceProp& props() const { return prop; }
    void select() const { CUDA_OK(cudaSetDevice(cuda_id)); }
    const stream_t& operator[](size_t i) const { return *streams[i % 3]; }
    void sync() const { for (auto& s : streams) s->sync(); }
};

const gpu_t& select_gpu(int id = 0);     // id == -1: the caller's current device
size_t ngpus();
const std::vector<const gpu_t*>& all_gpus();
const gpu_t& gpu_of_current_device();
