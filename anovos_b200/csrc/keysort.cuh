// Host driver of the LSD radix sort (sort.cu) for ONE caller-filled column of 64-bit keys.
// The caller writes n_rows keys to `buf[0]`; key_sort64 then runs the 64-bit tile histogram / totals / scan / scatter
// passes first_pass .. end_pass - 1 over them.  Every key is sorted: nothing is dropped and zero keys are not set aside
// (unlike the packing of anv_mode_distinct).  The passes are stable, so bytes below first_pass keep the order the keys
// arrived in.  The sorted keys end up in buf[*cur] (a device int, set by the scan kernels).
#pragma once
#include "common.cuh"

namespace anv {

struct KeySort64 {
  uint64_t* buf[2];
  const int* cur;   // [dev]
};

size_t key_sort64_workspace_bytes(int64_t n_rows);
// Carves the sort buffers out of `workspace` (the first key_sort64_workspace_bytes(n_rows) bytes).
void key_sort64_bind(void* workspace, int64_t n_rows, KeySort64* out);
int key_sort64(void* workspace, size_t workspace_bytes, int64_t n_rows, int first_pass, int end_pass, cudaStream_t st);

}  // namespace anv
