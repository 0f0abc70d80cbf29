// C-ABI plumbing: last-error string, version, device probe.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace masr {
static thread_local char g_err[512] = "";
void set_last_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
bool pdl_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("MASR_PDL");
        v = (e && e[0] == '0') ? 0 : 1;
    }
    return v == 1;
}
}  // namespace masr

extern "C" const char* masr_last_error(void) { return masr::g_err; }

extern "C" int masr_abi_version(void) { return MASR_ABI_VERSION; }

// Fails loudly (non-zero + message) unless the current device is a Hopper sm_90 part: the
// library carries sm_90a SASS only and has no fallback path.
extern "C" int masr_check_device(void) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) { masr::set_last_error("cudaGetDevice: %s", cudaGetErrorString(e)); return (int)e; }
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, dev);
    if (e != cudaSuccess) { masr::set_last_error("cudaGetDeviceProperties: %s", cudaGetErrorString(e)); return (int)e; }
    if (prop.major != 9 || prop.minor != 0) {
        masr::set_last_error("masr_b200 needs an sm_90 (H100) device, found sm_%d%d (%s)", prop.major, prop.minor, prop.name);
        return MASR_ERR_UNSUPPORTED_DEVICE;
    }
    return MASR_OK;
}
