// ia_host.h -- host-side error plumbing shared by the translation units of libia_b200.so
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>

#include "../../include/ia_b200.h"

char* ia_err_buf();  // thread-local, defined in ia_kernels.cu

inline int ia_set_err(int code, const char* fmt, const char* detail = "") {
    snprintf(ia_err_buf(), 512, fmt, detail);
    return code;
}
#define set_err ia_set_err
#define IA_CHECK_CUDA(expr)                                                                        \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) return ia_set_err(IA_ECUDA, #expr ": %s", cudaGetErrorString(_e)); \
    } while (0)
#define IA_REQUIRE(cond)                                                        \
    do {                                                                        \
        if (!(cond)) return ia_set_err(IA_EINVAL, "invalid argument: %s", #cond); \
    } while (0)

// Per-device caches (one process may drive several GPUs: function attributes and the SM count belong to a device)
constexpr int kMaxDevices = 64;
inline int current_device() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return -1;
    return dev;
}

inline int sm_count() {
    static int g_sm_count[kMaxDevices] = {};
    const int dev = current_device();
    if (dev < 0) return 0;
    int& c = g_sm_count[dev % kMaxDevices];
    if (!c) cudaDeviceGetAttribute(&c, cudaDevAttrMultiProcessorCount, dev);
    return c;
}

// "has the >48 KB shared-memory opt-in been applied to this kernel on the current device?"
struct PerDeviceFlag {
    bool done[kMaxDevices] = {};
    bool get() const { const int d = current_device(); return d >= 0 && done[d % kMaxDevices]; }
    void set() { const int d = current_device(); if (d >= 0) done[d % kMaxDevices] = true; }
};

// Opts Kernel into `bytes` of dynamic shared memory (above the default 48 KB) once per device.  The template takes the
// kernel itself, not its type, so that kernels of one signature (render_fwd_kernel<4> and <2>) each get their own flag.
template <auto Kernel>
inline int allow_dynamic_smem(int bytes) {
    static PerDeviceFlag done;
    if (!done.get()) {
        IA_CHECK_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        done.set();
    }
    return IA_OK;
}

