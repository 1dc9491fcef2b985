// ABI version, error string, device info.
#include <map>
#include <mutex>
#include <utility>
#include "common.cuh"

namespace nerrf {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int sm_count() {
    static int cached[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    int& c = cached[dev & 63];
    if (c == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) c = n;
        else return 132;
    }
    return c;
}

int set_max_dynamic_smem(const void* kernel, size_t bytes) {
    static std::mutex mu;
    static std::map<std::pair<int, const void*>, size_t> set;      // function attributes are per device
    int dev = 0;
    NERRF_CHECK_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(mu);
    size_t& cur = set[std::make_pair(dev, kernel)];
    if (cur >= bytes) return NERRF_OK;
    NERRF_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    cur = bytes;
    return NERRF_OK;
}

}  // namespace nerrf

extern "C" int nerrf_abi_version(void) { return NERRF_ABI_VERSION; }

extern "C" const char* nerrf_last_error(void) { return nerrf::g_err; }

extern "C" int nerrf_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) {
        cudaGetLastError();
        nerrf::set_error("no CUDA device");
        return NERRF_ERR_NODEVICE;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
        cudaGetLastError();
        nerrf::set_error("cudaGetDeviceProperties failed");
        return NERRF_ERR_NODEVICE;
    }
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    if (prop.major != 9 || prop.minor != 0) {
        nerrf::set_error("device is sm_%d%d; this library is built for sm_90a only", prop.major, prop.minor);
        return NERRF_ERR_NODEVICE;
    }
    return NERRF_OK;
}
