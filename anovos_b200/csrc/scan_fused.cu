// K1+K2 instantiation: moments and private-counter histogram in one read.
// Two kernels, same results bit for bit: the register-staged loop (default) and the cp.async-staged loop (ANV_FUSED_STAGED=1:
// null-free columns go through a thread-private shared-memory ring).  The ring hides load latency behind the thread's own
// next batches but costs more instructions per element; the register-staged loop is the default.
#include <stdlib.h>
#include "scan_impl.cuh"
namespace anv {
int launch_fused(ScanParams& P, size_t smem, cudaStream_t st) {
  const char* e = getenv("ANV_FUSED_STAGED");   // read per call (a test flips it between two calls of one process)
  const int staged = e ? atoi(e) : ANV_FUSED_STAGED_DEFAULT;
  // the ring needs ST_D * ST_CH * 4 KB behind the counters: fall back to register staging when it does not fit one CTA
  if (staged && smem + STAGE_BYTES + 16 <= 200 * 1024) return launch_scan<true, 0, false, true>(P, smem, st);
  return launch_scan<true, 0, false, false>(P, smem, st);
}
}  // namespace anv
