// common.cuh -- shared host/device helpers for libpvnet_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdint>
#include <cstdio>

#include "../../include/pvnet_b200.h"

namespace pvnet {

// thread-local error text + per-thread launch counter (defined in common.cu)
void set_error(const char *fmt, ...);
long long &launch_counter();
int sm_count();
// cudaFuncAttributeMaxDynamicSharedMemorySize is per (function, device): set it once for each pair
// (DataParallel-style callers drive several devices from one process)
cudaError_t ensure_max_smem(const void *func, int bytes);

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// bump allocator over the caller's workspace
struct Carver {
    char *base;
    size_t off = 0;
    explicit Carver(void *p) : base(static_cast<char *>(p)) {}
    template <typename T>
    T *take(size_t n)
    {
        off = align_up(off, 256);
        T *p = reinterpret_cast<T *>(base + off);
        off += n * sizeof(T);
        return p;
    }
};

}  // namespace pvnet

#define PV_CHECK_ARG(cond, ...)                \
    do {                                       \
        if (!(cond)) {                         \
            pvnet::set_error(__VA_ARGS__);     \
            return PVNET_E_INVALID;            \
        }                                      \
    } while (0)

#define PV_CUDA(call)                                                                      \
    do {                                                                                   \
        cudaError_t e_ = (call);                                                           \
        if (e_ != cudaSuccess) {                                                           \
            pvnet::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_),       \
                             __FILE__, __LINE__);                                          \
            return PVNET_E_CUDA;                                                           \
        }                                                                                  \
    } while (0)

// after every kernel launch: count it, surface launch-configuration errors
#define PV_LAUNCHED(name)                                                                  \
    do {                                                                                   \
        ++pvnet::launch_counter();                                                         \
        cudaError_t e_ = cudaGetLastError();                                               \
        if (e_ != cudaSuccess) {                                                           \
            pvnet::set_error("launch of %s failed: %s", name, cudaGetErrorString(e_));     \
            return PVNET_E_CUDA;                                                           \
        }                                                                                  \
    } while (0)
