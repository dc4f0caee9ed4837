// capi.cu -- error reporting, device info and library-level entry points of libesr_b200.so
#include "common.cuh"
#include <string>

namespace esr {

static thread_local std::string t_err;
std::atomic<long long> g_launches{0};

void set_error(const char *fmt, ...)
{
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    t_err = buf;
}

const DevInfo &dev_info()
{
    static DevInfo info = [] {
        DevInfo d{132, 232448};
        int dev = 0;
        if (cudaGetDevice(&dev) == cudaSuccess) {
            cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, dev);
            cudaDeviceGetAttribute(&d.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        }
        return d;
    }();
    return info;
}

} // namespace esr

extern "C" int esr_version(void) { return 100; }
extern "C" const char *esr_last_error(void) { return esr::t_err.c_str(); }
extern "C" int64_t esr_launch_count(void) { return (int64_t)esr::g_launches.load(); }
