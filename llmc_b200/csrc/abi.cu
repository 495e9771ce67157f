// abi.cu — version / error reporting of the C ABI (include/llmc_b200.h) and the launch
// bookkeeping every entry point shares.
#include <atomic>
#include <set>
#include <stdarg.h>
#include <string.h>
#include <utility>

#include "common.cuh"

namespace llmc {

static thread_local char g_last_error[512] = {0};

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}

static std::atomic<long long> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int opt_in_smem(const void* kernel, int bytes) {
  static std::mutex mutex;
  static std::set<std::pair<int, const void*>> done;
  int dev = 0;
  LLMC_CHECK_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> guard(mutex);
  if (done.count({dev, kernel})) return LLMC_OK;
  LLMC_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done.insert({dev, kernel});
  return LLMC_OK;
}

}  // namespace llmc

extern "C" long long llmc_b200_launch_count(void) {
  return llmc::g_launches.load(std::memory_order_relaxed);
}

extern "C" int llmc_b200_abi_version(void) { return LLMC_B200_ABI_VERSION; }

extern "C" const char* llmc_b200_error_string(int code) {
  switch (code) {
    case LLMC_OK: return "ok";
    case LLMC_EINVAL: return "invalid argument";
    case LLMC_EUNSUPPORTED: return "unsupported configuration";
    case LLMC_ECUDA: return "CUDA error";
    case LLMC_EALIGN: return "misaligned pointer or leading dimension";
    default: return "unknown error code";
  }
}

extern "C" const char* llmc_b200_last_error(void) { return llmc::g_last_error; }
