// Device enumeration: the reference's util/all_gpus.cpp:14-63 (gpus_t, select_gpu, ngpus,
// all_gpus) for this library.  Requires compute capability 9.0 (the kernels are built for
// sm_90a only, which loads on no other architecture); anything else is treated as "no device",
// there is no fallback path.
#include "gpu.cuh"

namespace {
struct gpus_t {
    std::vector<const gpu_t*> gpus;
    gpus_t()
    {
        int n = 0;
        if (cudaGetDeviceCount(&n) != cudaSuccess) { (void)cudaGetLastError(); return; }
        int prev = 0;
        (void)cudaGetDevice(&prev);
        for (int id = 0; id < n; id++) {
            cudaDeviceProp prop;
            if (cudaGetDeviceProperties(&prop, id) == cudaSuccess && prop.major == 9 && prop.minor == 0) {
                try { gpus.push_back(new gpu_t((int)gpus.size(), id)); } catch (const cuda_error&) {}
            }
        }
        (void)cudaSetDevice(prev);
    }
    static gpus_t& all() { static gpus_t g; return g; }
};
}  // namespace

const std::vector<const gpu_t*>& all_gpus() { return gpus_t::all().gpus; }
size_t ngpus() { return all_gpus().size(); }

const gpu_t& gpu_of_current_device()
{
    auto& gpus = all_gpus();
    if (gpus.empty()) CUDA_OK(cudaErrorNoDevice);
    int cid;
    CUDA_OK(cudaGetDevice(&cid));
    for (auto* g : gpus)
        if (g->cid() == cid) return *g;
    throw cuda_error(-(int)cudaErrorInvalidDevice, "current CUDA device is not an H100-class (sm_90) device");
}

const gpu_t& select_gpu(int id)
{
    auto& gpus = all_gpus();
    if (gpus.empty()) CUDA_OK(cudaErrorNoDevice);
    if (id == -1) return gpu_of_current_device();
    if (id < 0 || (size_t)id >= gpus.size())
        throw cuda_error(-(int)cudaErrorInvalidDevice, "select_gpu: no such device");
    gpus[id]->select();
    return *gpus[id];
}
