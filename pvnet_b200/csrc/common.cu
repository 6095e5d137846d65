// common.cu -- error string, launch counter, device queries.
#include "common.cuh"

#include <cstring>
#include <mutex>
#include <set>
#include <utility>

namespace pvnet {

static thread_local char g_err[512] = "";
static thread_local long long g_launches = 0;

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

long long &launch_counter() { return g_launches; }

int sm_count()
{
    static thread_local int cached_dev = -1, cached = 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 148;
    if (dev != cached_dev) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 148;
        cached = n;
        cached_dev = dev;
    }
    return cached;
}

cudaError_t ensure_max_smem(const void *func, int bytes)
{
    static std::mutex mu;
    static std::set<std::pair<const void *, int>> done;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lock(mu);
    if (done.count({func, dev})) return cudaSuccess;
    e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) done.insert({func, dev});
    return e;
}

}  // namespace pvnet

extern "C" {

const char *pvnet_last_error(void) { return pvnet::g_err; }
int pvnet_version(void) { return 3; }
long long pvnet_launch_count(void) { return pvnet::launch_counter(); }
void pvnet_launch_count_reset(void) { pvnet::launch_counter() = 0; }

}  // extern "C"
