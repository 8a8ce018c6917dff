// ABI housekeeping: version, thread-local error string, device probes.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace rl {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
// Upper bound on the CTAs a persistent network kernel launches (0 = one per SM).  Two streams that both launch
// whole-GPU persistent grids serialise; capping each side lets the actor's and the learner's kernels share the SMs.
static int g_sm_limit = 0;
int effective_sms(int sms) { return (g_sm_limit > 0 && g_sm_limit < sms) ? g_sm_limit : sms; }
// Programmatic dependent launch of the actor-chain kernels (common.cuh: launch_chain / pdl_wait).  OFF by default:
// early-resident CTAs of the next kernel hold SMs that the other stream's kernels of a pipelined step could use.
static int g_pdl = 0;
int pdl_enabled() { return g_pdl; }
}  // namespace rl

extern "C" int rl_debug_set_pdl(int enable) {
  rl::g_pdl = enable ? 1 : 0;
  return RL_OK;
}

extern "C" int rl_set_sm_limit(int max_ctas) {
  if (max_ctas < 0) {
    rl::set_error("rl_set_sm_limit: %d < 0", max_ctas);
    return RL_ERR_BAD_ARG;
  }
  rl::g_sm_limit = max_ctas;
  return RL_OK;
}

extern "C" int rl_abi_version(void) { return 1; }
extern "C" const char* rl_last_error(void) { return rl::g_err; }
extern "C" int rl_device_sm_count(int device) {
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) {
    rl::set_error("rl_device_sm_count: %s", cudaGetErrorString(cudaGetLastError()));
    return RL_ERR_CUDA;
  }
  return n;
}
