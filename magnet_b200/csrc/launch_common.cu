// Host helpers shared by the launchers: SM count, the driver's tensor-map encoder and the work-slot tickets.
#include "launchers.h"

namespace magnet {

int sm_count(int dev) {
  static int cached[64] = {0};
  int& c = cached[dev & 63];
  if (c == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    c = n;
  }
  return c;
}

EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      f = nullptr;
    return reinterpret_cast<EncodeTiledFn>(f);
  }();
  return fn;
}

int work_slot(SlotTickets& tickets, cudaStream_t st) {
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cap) != cudaSuccess) cap = cudaStreamCaptureStatusNone;
  return cap == cudaStreamCaptureStatusActive ? WORK_SLOTS / 2 + (int)(tickets.captured.fetch_add(1) % (WORK_SLOTS / 2))
                                              : (int)(tickets.eager.fetch_add(1) % (WORK_SLOTS / 2));
}

}  // namespace magnet
