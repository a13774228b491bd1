// Library bookkeeping: version, status strings, last-error text, launch counter.
#include "common.cuh"

namespace hd {
std::atomic<long long> g_launches{0};
static thread_local char t_err[512] = "";

void set_last_error(const char *what, cudaError_t e) {
  snprintf(t_err, sizeof(t_err), "%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
}
void set_last_error_text(const char *what) { snprintf(t_err, sizeof(t_err), "%s", what); }
}  // namespace hd

extern "C" {

int hd_version(void) { return 107; }

const char *hd_status_string(int s) {
  switch (s) {
    case HD_OK: return "ok";
    case HD_ERR_INVALID: return "invalid argument";
    case HD_ERR_WORKSPACE: return "workspace too small";
    case HD_ERR_CUDA: return "cuda error";
    case HD_ERR_UNSUPPORTED: return "unsupported device or implementation";
    default: return "unknown status";
  }
}

const char *hd_last_error(void) { return hd::t_err; }
long long hd_launch_count(void) { return hd::g_launches.load(); }
void hd_launch_count_reset(void) { hd::g_launches.store(0); }

}  // extern "C"
