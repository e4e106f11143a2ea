// Misc C-ABI entry points (include/sppark_b200.h): device probing, error-message ownership,
// introspection.  Reference: util/all_gpus.cpp:65-86.
#include "util/gpu.cuh"

std::atomic<uint64_t> g_launch_count{0};

extern "C" int cuda_available(void)
{
    try { return ngpus() != 0; } catch (...) { return 0; }
}

extern "C" void drop_error_message(char* msg) { free(msg); }

extern "C" size_t sppark_b200_ngpus(void)
{
    try { return ngpus(); } catch (...) { return 0; }
}

extern "C" int sppark_b200_sm_count(int device_id)
{
    try { return select_gpu(device_id).sm_count(); } catch (...) { return -1; }
}

extern "C" const char* sppark_b200_version(void) { return "sppark_b200 0.1 (sm_90a)"; }

extern "C" uint64_t sppark_b200_launch_count(void) { return g_launch_count.load(); }

phase_profile_t g_profile;

extern "C" void sppark_b200_profile_enable(int on) { g_profile.enabled = on != 0; g_profile.reset(); }

// writes up to `cap` (name, ms) pairs for the phases of the last profiled call; returns count.
// ms[i] is the time from mark i to mark i+1.  Call after synchronising the stream.
extern "C" int sppark_b200_profile_read(const char** names, float* ms, int cap)
{
    int k = 0;
    for (int i = 0; i + 1 < g_profile.n && k < cap; i++, k++) {
        float t = 0;
        if (cudaEventElapsedTime(&t, g_profile.ev[i], g_profile.ev[i + 1]) != cudaSuccess) t = -1;
        names[k] = g_profile.name[i];
        ms[k] = t;
    }
    return k;
}

// ---- gpu_ptr_t: reference-counted device allocation handed across the FFI -------------------
// Same ABI as the reference (util/gpu_t.cuh:268-316, util/all_gpus.cpp:69-79; Rust
// `Gpu_Ptr<T>` is one pointer-sized word, rust/src/lib.rs:62-97): the handle points at
// {device pointer, atomic reference count, owning device}; the last drop frees the memory.
struct gpu_ptr_inner {
    void* ptr;
    std::atomic<size_t> ref_cnt;
    int real_id;
};
static gpu_ptr_inner* inner_of(const gpu_ptr_t* ref)
{   return ref ? static_cast<gpu_ptr_inner*>(ref->inner) : nullptr;   }

extern "C" void drop_gpu_ptr_t(gpu_ptr_t* ref)
{
    gpu_ptr_inner* in = inner_of(ref);
    if (in && in->ref_cnt.fetch_sub(1, std::memory_order_seq_cst) == 1) {
        int cur = 0;
        (void)cudaGetDevice(&cur);
        if (cur != in->real_id) (void)cudaSetDevice(in->real_id);
        (void)cudaFree(in->ptr);
        if (cur != in->real_id) (void)cudaSetDevice(cur);
        delete in;
    }
    if (ref) ref->inner = nullptr;
}

extern "C" gpu_ptr_t clone_gpu_ptr_t(const gpu_ptr_t* ref)
{
    gpu_ptr_inner* in = inner_of(ref);
    if (in) in->ref_cnt.fetch_add(1, std::memory_order_relaxed);
    return gpu_ptr_t{in};
}

// allocate `bytes` on the current device; {NULL} on failure
extern "C" gpu_ptr_t sppark_b200_gpu_ptr_alloc(size_t bytes)
{
    void* p = nullptr;
    if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess) {
        (void)cudaGetLastError();
        return gpu_ptr_t{nullptr};
    }
    auto* in = new gpu_ptr_inner;
    in->ptr = p;
    in->ref_cnt.store(1);
    in->real_id = 0;
    (void)cudaGetDevice(&in->real_id);
    return gpu_ptr_t{in};
}

extern "C" void* sppark_b200_gpu_ptr_get(const gpu_ptr_t* ref)
{   gpu_ptr_inner* in = inner_of(ref); return in ? in->ptr : nullptr;   }

extern "C" size_t sppark_b200_gpu_ptr_refs(const gpu_ptr_t* ref)
{   gpu_ptr_inner* in = inner_of(ref); return in ? in->ref_cnt.load() : 0;   }

// ---- peer buffers for the fused NTT exchange (ntt/ntt_plan.hpp: make_slab_plan) -------------
// One process per GPU: each rank allocates its receive buffer with cudaMalloc, exports a CUDA IPC
// handle (64 bytes, exchanged by the caller over its process group), and maps the other ranks'
// buffers; stores to the mapped pointers travel over NVLink / NVSwitch.
static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");

extern "C" RustError sppark_b200_peer_alloc(size_t bytes, void** d_ptr, void* ipc_handle)
{
    try {
        if (d_ptr == nullptr || ipc_handle == nullptr) throw cuda_error(-(int)cudaErrorInvalidValue, "peer_alloc: null argument");
        (void)gpu_of_current_device();
        CUDA_OK(cudaMalloc(d_ptr, bytes ? bytes : 1));
        cudaIpcMemHandle_t h;
        cudaError_t e = cudaIpcGetMemHandle(&h, *d_ptr);
        if (e != cudaSuccess) { (void)cudaFree(*d_ptr); *d_ptr = nullptr; CUDA_OK(e); }
        memcpy(ipc_handle, &h, sizeof(h));
    } catch (const cuda_error& e) {
        return rust_err(e.code(), e.what());
    }
    return rust_ok();
}

extern "C" RustError sppark_b200_peer_open(const void* ipc_handle, void** d_ptr)
{
    try {
        if (d_ptr == nullptr || ipc_handle == nullptr) throw cuda_error(-(int)cudaErrorInvalidValue, "peer_open: null argument");
        (void)gpu_of_current_device();
        cudaIpcMemHandle_t h;
        memcpy(&h, ipc_handle, sizeof(h));
        CUDA_OK(cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    } catch (const cuda_error& e) {
        return rust_err(e.code(), e.what());
    }
    return rust_ok();
}

extern "C" RustError sppark_b200_peer_close(void* d_ptr)
{
    cudaError_t e = cudaIpcCloseMemHandle(d_ptr);
    return e == cudaSuccess ? rust_ok() : rust_err(-(int)e, cudaGetErrorString(e));
}

extern "C" RustError sppark_b200_peer_free(void* d_ptr)
{
    cudaError_t e = cudaFree(d_ptr);
    return e == cudaSuccess ? rust_ok() : rust_err(-(int)e, cudaGetErrorString(e));
}
