// Error plumbing and per-device launch state shared by the C-ABI translation units.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdio>
#include <string>

#include "../../include/rf_b200.h"

void rf_set_error(const std::string& msg);
int rf_fail(int code, const std::string& msg);

#define RF_CUDA_TRY(expr)                                                                      \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess)                                                                 \
            return rf_fail(RF_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));   \
    } while (0)

#define RF_CUDA_LAUNCH_CHECK(name)                                                             \
    do {                                                                                       \
        cudaError_t _e = cudaGetLastError();                                                   \
        if (_e != cudaSuccess)                                                                 \
            return rf_fail(RF_ERR_CUDA, std::string("launch ") + name + ": " +                 \
                                            cudaGetErrorString(_e));                           \
    } while (0)


// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a PER-DEVICE property of a kernel: remember it per (call site,
// device) so that a process driving several GPUs (ADVICE r1) sets it on each of them.  Up to 64 devices.
struct rf_dev_once {
    std::atomic<unsigned long long> done{0};
};
template <class F>
inline cudaError_t rf_set_smem_once(rf_dev_once& o, F* func, int bytes) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const unsigned long long bit = 1ull << (dev & 63);
    if (o.done.load(std::memory_order_acquire) & bit) return cudaSuccess;
    e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) o.done.fetch_or(bit, std::memory_order_release);
    return e;
}

// SM count of the current device, cached per device like rf_set_smem_once (up to 64 devices); 132, the H100 SXM's count,
// if the query fails.  Launch geometries scale with it.
inline int rf_num_sms() {
    static std::atomic<int> cached[64];
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    std::atomic<int>& c = cached[dev & 63];
    if ((n = c.load(std::memory_order_relaxed))) return n;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
    c.store(n, std::memory_order_relaxed);
    return n;
}


// ---------------------------------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  A CFG UNet evaluation is ~440 dependent launches; with the attribute below the
// next kernel's CTAs are scheduled as soon as every CTA of the current one has passed rf_pdl_trigger(), run their prologue
// (barrier init, descriptor prefetch) and then block in rf_pdl_wait() until the current grid has completed and its
// writes are visible.  Rules that keep this safe:
//   * a kernel launched through RF_LAUNCH_PDL executes rf_pdl_wait() in EVERY thread before its first global-memory access
//     (reads of the producer's output and writes that could overtake the producer's reads alike);
//   * everything else is launched the ordinary way and therefore still waits for full completion of its predecessor.
// Early-resident dependents hide launch latency when the kernels are short, but at large batches they only take
// resources from the tail of the running grid.  Hence the default mode: the attribute goes on launches that cannot fill
// the GPU anyway (`small`: a couple of waves at most — the single-request regime) and stays off otherwise.
// RF_PDL in the environment: 0 = never, 1 = small launches (default), 2 = every instrumented launch.  Without the attribute
// the device instructions are no-ops.
#include <cstdlib>
inline int rf_pdl_mode() {
    static const int mode = [] {
        const char* e = std::getenv("RF_PDL");
        return e ? std::atoi(e) : 1;
    }();
    return mode;
}
inline bool rf_pdl_use(bool small) { return rf_pdl_mode() >= 2 || (rf_pdl_mode() == 1 && small); }
#if defined(__CUDACC__)
__device__ __forceinline__ void rf_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void rf_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#endif
// kernel may be a template-id in parentheses; extra attributes (cluster dimension) go in front of the PDL one
#define RF_LAUNCH_PDL_ATTRS(name, kernel, grid, block, smem, st, small, attr_arr, n_attr, ...)                                   \
    do {                                                                                                             \
        cudaLaunchConfig_t _cfg = {};                                                                                \
        _cfg.gridDim = (grid);                                                                                       \
        _cfg.blockDim = (block);                                                                                     \
        _cfg.dynamicSmemBytes = (smem);                                                                              \
        _cfg.stream = (st);                                                                                          \
        (attr_arr)[n_attr].id = cudaLaunchAttributeProgrammaticStreamSerialization;                                      \
        (attr_arr)[n_attr].val.programmaticStreamSerializationAllowed = 1;                                               \
        _cfg.attrs = (attr_arr);                                                                                        \
        _cfg.numAttrs = (n_attr) + (rf_pdl_use(small) ? 1 : 0);                                                        \
        const cudaError_t _le = cudaLaunchKernelEx(&_cfg, kernel, __VA_ARGS__);                                      \
        if (_le != cudaSuccess) return rf_fail(RF_ERR_CUDA, std::string("launch ") + name + ": " + cudaGetErrorString(_le)); \
    } while (0)
#define RF_LAUNCH_PDL(name, kernel, grid, block, smem, st, small, ...)                                                       \
    do {                                                                                                             \
        cudaLaunchAttribute _attr[1];                                                                                \
        RF_LAUNCH_PDL_ATTRS(name, kernel, grid, block, smem, st, small, _attr, 0, __VA_ARGS__);                             \
    } while (0)
