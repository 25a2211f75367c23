// Host side of the column scan: tile sizing, the finalize (Pebay merge) kernel and the C ABI.
#include "scan_impl.cuh"

namespace anv {

// One warp per column: lane-strided sequential Pebay merge, then a shuffle tree.
__global__ void __launch_bounds__(32) finalize_moments(const Partial* partials, int tiles_per_col, anv_moments_t* out) {
  const int c = blockIdx.x, lane = threadIdx.x;
  const Partial* p = partials + (size_t)c * tiles_per_col;
  Central acc{0, 0, 0, 0, 0};
  int64_t n = 0, nz = 0;
  double mn = INFINITY, mx = -INFINITY;
  for (int t = lane; t < tiles_per_col; t += 32) {
    const Partial q = p[t];
    if (q.n > 0) {
      acc = merge_central(acc, Central{(double)q.n, q.mean, q.m2, q.m3, q.m4});
      mn = fmin(mn, q.mn);
      mx = fmax(mx, q.mx);
    }
    n += q.n;
    nz += q.nz;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Central b;
    b.n = shfl_down_d(acc.n, o); b.mean = shfl_down_d(acc.mean, o);
    b.m2 = shfl_down_d(acc.m2, o); b.m3 = shfl_down_d(acc.m3, o); b.m4 = shfl_down_d(acc.m4, o);
    acc = merge_central(acc, b);
    mn = fmin(mn, shfl_down_d(mn, o));
    mx = fmax(mx, shfl_down_d(mx, o));
    n += shfl_down_ll(n, o);
    nz += shfl_down_ll(nz, o);
  }
  if (lane == 0) {
    anv_moments_t r;
    r.n_valid = n; r.n_nonzero = nz;
    if (n > 0) {
      r.mean = acc.mean; r.m2 = acc.m2; r.m3 = acc.m3; r.m4 = acc.m4;
      // min / max skip NaN; with nothing but NaN they are NaN (as the order statistics are), not the start values
      if (mn > mx) mn = mx = nan("");
      r.min = mn; r.max = mx;
    } else { r.min = r.max = r.mean = nan(""); r.m2 = r.m3 = r.m4 = 0.0; }
    out[c] = r;
  }
}

int pick_tile_rows(int64_t n_rows, int n_cols) {
  // >= ~8 tiles per SM across the launch, tile in [16Ki, 256Ki] rows, multiple of 1024
  int sms = 132, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int64_t want_tiles = (int64_t)sms * 8;
  int64_t per_col = (want_tiles + n_cols - 1) / (n_cols > 0 ? n_cols : 1);
  int64_t tr = per_col > 0 ? n_rows / per_col : n_rows;
  int64_t t = 16384;
  while (t < tr && t < 262144) t <<= 1;
  return (int)t;
}

size_t hist_smem(int count_stride, int* path, int* thr_slots, bool codes) {
  int nb = count_stride - 1, p2 = 2;
  while (p2 < nb) p2 <<= 1;
  *thr_slots = codes ? 2 : p2 + 2;  // dictionary codes need no thresholds
  size_t thr = (size_t)(*thr_slots) * 8;
  if (count_stride <= 40) { *path = 0; return thr + 2 * (size_t)count_stride * ANV_BLOCK * 4; }  // counters + per-thread threshold replica
  if (count_stride <= 10240) { *path = 1; return thr + (size_t)count_stride * 4; }
  *path = 2;
  return thr;
}

int check_common(const void* cols, int n_cols, int64_t n_rows) {
  if (n_cols < 0 || n_rows < 0) { set_error("negative n_cols / n_rows"); return ANV_ERR_INVALID; }
  if (n_cols > ANV_MAX_LAUNCH_COLS) { set_error("n_cols > %d: split the frame into column blocks", ANV_MAX_LAUNCH_COLS); return ANV_ERR_UNSUPPORTED; }
  if (n_cols > 0 && !cols) { set_error("cols is NULL"); return ANV_ERR_INVALID; }
  return ANV_OK;
}

static void base_params(ScanParams& P, const anv_column_t* cols, int n_cols, int64_t n_rows) {
  P.cols = cols; P.n_cols = n_cols; P.n_rows = n_rows;
  P.tile_rows = pick_tile_rows(n_rows > 0 ? n_rows : 1, n_cols);
  P.tiles_per_col = n_rows ? (int)((n_rows + P.tile_rows - 1) / P.tile_rows) : 0;
}

}  // namespace anv

using namespace anv;

extern "C" size_t anv_moments_workspace_bytes(int n_cols, int64_t n_rows) {
  if (n_cols <= 0 || n_rows <= 0) return 64;
  const int tr = pick_tile_rows(n_rows, n_cols);
  const int64_t tiles = (n_rows + tr - 1) / tr;
  return (size_t)tiles * (size_t)n_cols * sizeof(Partial) + 64;
}

extern "C" int anv_moments(const anv_column_t* cols, int n_cols, int64_t n_rows, anv_moments_t* out, void* workspace,
                           size_t workspace_bytes, void* stream) {
  if (int e = check_common(cols, n_cols, n_rows)) return e;
  if (n_cols == 0) return ANV_OK;
  if (!out) { set_error("out is NULL"); return ANV_ERR_INVALID; }
  if (workspace_bytes < anv_moments_workspace_bytes(n_cols, n_rows) || !workspace) {
    set_error("anv_moments: workspace too small (%zu < %zu)", workspace_bytes, anv_moments_workspace_bytes(n_cols, n_rows));
    return ANV_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  ScanParams P{};
  base_params(P, cols, n_cols, n_rows);
  P.partials = reinterpret_cast<Partial*>(workspace);
  if (int e = launch_mom(P, st)) return e;
  finalize_moments<<<n_cols, 32, 0, st>>>(P.partials, P.tiles_per_col, out);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

extern "C" int anv_hist(const anv_column_t* cols, const anv_binspec_t* specs, const void* cuts, int n_cols, int64_t n_rows,
                        uint64_t* counts, int count_stride, void* stream) {
  if (int e = check_common(cols, n_cols, n_rows)) return e;
  if (n_cols == 0) return ANV_OK;
  if (!specs || !counts || count_stride < 2) { set_error("anv_hist: bad specs/counts/count_stride"); return ANV_ERR_INVALID; }
  if (count_stride > ANV_MAX_BINS + 1) {
    set_error("anv_hist: more than %d bins per column is not supported", ANV_MAX_BINS);
    return ANV_ERR_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  ANV_CUDA(cudaMemsetAsync(counts, 0, (size_t)n_cols * count_stride * sizeof(uint64_t), st));
  ScanParams P{};
  base_params(P, cols, n_cols, n_rows);
  P.specs = specs; P.cuts = reinterpret_cast<const uint64_t*>(cuts);
  P.counts = reinterpret_cast<unsigned long long*>(counts); P.count_stride = count_stride;
  int path = 0;
  size_t smem = hist_smem(count_stride, &path, &P.thr_slots);
  return launch_hist(P, path, smem, st);
}

extern "C" int anv_hist_codes(const anv_column_t* cols, const int32_t* cardinality, int n_cols, int64_t n_rows,
                              uint64_t* counts, int count_stride, void* stream) {
  if (int e = check_common(cols, n_cols, n_rows)) return e;
  if (n_cols == 0) return ANV_OK;
  if (!cardinality || !counts || count_stride < 2) { set_error("anv_hist_codes: bad arguments"); return ANV_ERR_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  ANV_CUDA(cudaMemsetAsync(counts, 0, (size_t)n_cols * count_stride * sizeof(uint64_t), st));
  ScanParams P{};
  base_params(P, cols, n_cols, n_rows);
  P.card = cardinality;
  P.counts = reinterpret_cast<unsigned long long*>(counts); P.count_stride = count_stride;
  int path = 0;
  size_t smem = hist_smem(count_stride, &path, &P.thr_slots, true);
  return launch_hist(P, path, smem, st);
}

extern "C" int anv_moments_hist(const anv_column_t* cols, const anv_binspec_t* specs, const void* cuts, int n_cols,
                                int64_t n_rows, anv_moments_t* out, uint64_t* counts, int count_stride, void* workspace,
                                size_t workspace_bytes, void* stream) {
  if (int e = check_common(cols, n_cols, n_rows)) return e;
  if (n_cols == 0) return ANV_OK;
  if (!specs || !counts || !out || count_stride < 2) { set_error("anv_moments_hist: bad arguments"); return ANV_ERR_INVALID; }
  if (count_stride > ANV_MAX_BINS + 1) {
    set_error("anv_moments_hist: more than %d bins per column is not supported", ANV_MAX_BINS);
    return ANV_ERR_UNSUPPORTED;
  }
  if (workspace_bytes < anv_moments_workspace_bytes(n_cols, n_rows) || !workspace) {
    set_error("anv_moments_hist: workspace too small");
    return ANV_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  ANV_CUDA(cudaMemsetAsync(counts, 0, (size_t)n_cols * count_stride * sizeof(uint64_t), st));
  ScanParams P{};
  base_params(P, cols, n_cols, n_rows);
  P.partials = reinterpret_cast<Partial*>(workspace);
  P.specs = specs; P.cuts = reinterpret_cast<const uint64_t*>(cuts);
  P.counts = reinterpret_cast<unsigned long long*>(counts); P.count_stride = count_stride;
  int path = 0;
  size_t smem = hist_smem(count_stride, &path, &P.thr_slots);
  if (path == 0) {
    if (int e = launch_fused(P, smem, st)) return e;
  } else {  // wide histograms: two kernels (the fused variant only pays off with private counters)
    if (int e = launch_mom(P, st)) return e;
    if (int e = launch_hist(P, path, smem, st)) return e;
  }
  finalize_moments<<<n_cols, 32, 0, st>>>(P.partials, P.tiles_per_col, out);
  ANV_CUDA(cudaGetLastError());
  return ANV_OK;
}

extern "C" int anv_bin_assign(const anv_column_t* cols, const anv_binspec_t* specs, const void* cuts, int n_cols,
                              int64_t n_rows, int max_bins, int32_t* out_bins, int64_t out_stride, void* stream) {
  if (int e = check_common(cols, n_cols, n_rows)) return e;
  if (n_cols == 0) return ANV_OK;
  if (!specs || !out_bins || out_stride < n_rows || (out_stride & 3) || max_bins < 2) {
    set_error("anv_bin_assign: bad arguments (out_stride must be >= n_rows and a multiple of 4; max_bins >= 2)");
    return ANV_ERR_INVALID;
  }
  if (max_bins > ANV_MAX_BINS) {
    set_error("anv_bin_assign: more than %d bins per column is not supported", ANV_MAX_BINS);
    return ANV_ERR_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  ScanParams P{};
  base_params(P, cols, n_cols, n_rows);
  P.specs = specs; P.cuts = reinterpret_cast<const uint64_t*>(cuts);
  P.out_bins = out_bins; P.out_stride = out_stride;
  int path = 0;
  hist_smem(max_bins + 1, &path, &P.thr_slots);
  return launch_assign(P, (size_t)P.thr_slots * 8, st);
}
