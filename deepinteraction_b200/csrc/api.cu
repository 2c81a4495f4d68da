// Error reporting and version entry points of libdi_b200 (see include/di_b200.h).
#include "common.cuh"
#include <stdarg.h>

static thread_local char g_err[512] = "";

void di_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" {

const char* di_last_error(void) { return g_err; }

int di_version(void) { return 100; }

// Compute capability the library was built for (major*10+minor); the kernels use sm_90a only.
int di_built_arch(void) { return 90; }

}  // extern "C"
