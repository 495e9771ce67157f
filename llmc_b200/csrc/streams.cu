// streams.cu — the per-device side streams of the look-ahead schedules (see common.cuh).
#include "common.cuh"

namespace llmc {

int side_streams(int64_t n_events, SideStreams** out) {
  constexpr int kMaxDev = 64;
  static std::mutex mutex;
  static SideStreams of[kMaxDev];
  static bool created[kMaxDev];
  int dev = 0;
  LLMC_CHECK_CUDA(cudaGetDevice(&dev));
  dev &= kMaxDev - 1;
  std::lock_guard<std::mutex> guard(mutex);
  SideStreams& s = of[dev];
  if (!created[dev]) {
    int least = 0, greatest = 0;
    LLMC_CHECK_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
    const int mid = (greatest < least) ? greatest + 1 : greatest;
    const int priority[kNumSideStreams] = {greatest, mid, least, least};
    for (int i = 0; i < kNumSideStreams; ++i) {
      LLMC_CHECK_CUDA(cudaStreamCreateWithPriority(&s.stream[i], cudaStreamNonBlocking, priority[i]));
      LLMC_CHECK_CUDA(cudaEventCreateWithFlags(&s.join_ev[i], cudaEventDisableTiming));
    }
    LLMC_CHECK_CUDA(cudaEventCreateWithFlags(&s.fork_ev, cudaEventDisableTiming));
    created[dev] = true;
  }
  for (std::vector<cudaEvent_t>& v : s.ev) {
    while (static_cast<int64_t>(v.size()) < n_events) {
      cudaEvent_t e;
      LLMC_CHECK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      v.push_back(e);
    }
  }
  *out = &s;
  return LLMC_OK;
}

int SideStreams::fork(cudaStream_t st, std::initializer_list<SideStream> to) {
  LLMC_CHECK_CUDA(cudaEventRecord(fork_ev, st));
  for (SideStream r : to) LLMC_CHECK_CUDA(cudaStreamWaitEvent(stream[r], fork_ev, 0));
  return LLMC_OK;
}

int SideStreams::join(cudaStream_t st, std::initializer_list<SideStream> from) {
  for (SideStream r : from) {
    LLMC_CHECK_CUDA(cudaEventRecord(join_ev[r], stream[r]));
    LLMC_CHECK_CUDA(cudaStreamWaitEvent(st, join_ev[r], 0));
  }
  return LLMC_OK;
}

}  // namespace llmc
