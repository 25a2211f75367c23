/*
 * anovos_b200.h - C ABI of libanovos_b200.so: the H100 (sm_90a) kernels behind the
 * Anovos stats_generator / attribute_binning / drift_detector hot path.
 *
 * The reference (anovos/anovos v1.1.0) has NO native / FFI interface: its boundary is the
 * Python module API that workflow.py resolves by name (SURVEY.md 8b).  Each entry point
 * below therefore cites the reference Python code whose work it replaces (paths relative
 * to /root/reference/src/main/anovos); INTEGRATION.md shows the ctypes binding a
 * maintainer would add on the reference side.
 *
 * Conventions
 *  - Plain C: pointers + sizes, no C++ / torch types.  Every function returns 0 on
 *    success or a negative anv_status; anv_last_error() gives a thread-local message.
 *  - The CALLER owns every buffer (columns, outputs, workspaces).  The library allocates
 *    nothing persistent, keeps no global state, is re-entrant per stream and never
 *    synchronises the device (all work is enqueued on `stream`).
 *  - Pointers marked [dev] are device pointers, [host] host pointers.
 *  - Columns are column-major: one contiguous array per column, 16-byte aligned,
 *    n_rows elements.  `validity` is an Arrow validity bitmap (LSB-first, 1 = valid)
 *    readable as ceil(n_rows/32) 32-bit words, or NULL when the column has no nulls.
 */
#ifndef ANOVOS_B200_H
#define ANOVOS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ANV_VERSION 100 /* 0.1.0 */

/* Most column passes launch one grid row per column (gridDim.y <= 65535): the entry points that take anv_column_t
 * descriptors reject more columns per call with ANV_ERR_UNSUPPORTED, and a caller splits a wider frame into column
 * blocks of at most this many (every per-column result is independent of the other columns of the call). */
#define ANV_MAX_LAUNCH_COLS 65535

typedef enum {
  ANV_OK = 0,
  ANV_ERR_INVALID = -1,   /* bad argument (null pointer, misaligned column, bad dtype ...) */
  ANV_ERR_WORKSPACE = -2, /* workspace too small: call the matching *_workspace_bytes */
  ANV_ERR_CUDA = -3,      /* a CUDA runtime call failed; see anv_last_error() */
  ANV_ERR_UNSUPPORTED = -4
} anv_status;

typedef enum { ANV_F32 = 0, ANV_F64 = 1, ANV_I32 = 2, ANV_I64 = 3 } anv_dtype;

/* One input column.  Spark dtype mapping (shared/utils.py:64-72): float->F32,
 * double->F64, int->I32, bigint/long->I64; dictionary codes of string columns -> I32. */
typedef struct {
  const void* data;         /* [dev] n_rows elements, 16-byte aligned */
  const uint32_t* validity; /* [dev] Arrow bitmap words or NULL */
  int32_t dtype;            /* anv_dtype */
  int32_t reserved;
} anv_column_t;

/* Per-column result of the fused moments pass.  All floating-point aggregates are
 * computed in float64 on double(x), like Spark (SURVEY.md 8a semantics item 1).
 * m2..m4 are CENTRAL power sums  sum (x-mean)^k  over the non-null values. */
typedef struct {
  int64_t n_valid;   /* count(col): non-null rows      (stats_generator.py:163,310) */
  int64_t n_nonzero; /* MLlib numNonzeros after null->0 (stats_generator.py:240-241) */
  double min, max;   /* NaN when n_valid == 0           (stats_generator.py:813,908; transformers.py:217-219) */
  double mean;       /* avg(double(x))                  (stats_generator.py:488,813) */
  double m2, m3, m4; /* -> stddev_samp / skewness / kurtosis (stats_generator.py:813,993) */
} anv_moments_t;

/* Per-column binning model: bucket_label (transformers.py:248-271) assigns
 * bin = 1 + #(cutoffs strictly below v), null -> slot 0.
 * The n_bins-1 cutoffs are given as NATIVE-TYPE thresholds (8 bytes per slot in
 * `cuts`, value in the low bytes): for a float32 column  double(v) <= c  <=>
 * v <= rounddown_f32(c), for int columns v <= floor(c): the comparison is exact
 * without any FP64 work in the kernel.  mode 1 (equal_range) additionally supplies
 * lo / inv_w so the kernel can guess the bin with one FMA and fix it up with a
 * single exact threshold compare. */
typedef struct {
  int32_t n_bins;     /* bin ids 1..n_bins; counts slot 0 = null rows */
  int32_t mode;       /* 0 = generic sorted cutoffs (binary search), 1 = equal_range */
  double lo;          /* mode 1: source min                       (transformers.py:229) */
  double inv_w;       /* mode 1: bin_size / (max - min)                                 */
  int64_t cut_offset; /* first threshold slot of this column in `cuts`                  */
} anv_binspec_t;

/* Drift metrics of one column (drift_detector.py:273-335; no rounding). */
typedef struct {
  double psi, hd, jsd, ks;
  int32_t n_rows; /* rows of the (p,q) table that were reduced; 0 => metrics are NaN */
  int32_t reserved;
} anv_drift_t;

/* ---- library ------------------------------------------------------------------- */
int anv_version(void);
/* sha1 of the sources the binary was built from (build-time define); "unknown" for an ad-hoc build. */
const char* anv_source_hash(void);
const char* anv_last_error(void);
/* sm_count / cc_major / cc_minor / total_mem of the CURRENT device. */
int anv_device_info(int* sm_count, int* cc_major, int* cc_minor, size_t* total_mem);

/* ---- K1: fused moments pass  (replaces the Spark jobs behind stats_generator.py:
 *      163,240-241,310,488,813,908,993 and transformers.py:217-219, stability.py:241-243)
 * One streaming read of every column: n_valid, n_nonzero, min, max and shifted power
 * sums in FP64 per (column, row-tile), then a deterministic Pebay merge per column.
 * cols [dev] n_cols descriptors; out [dev] n_cols results. */
size_t anv_moments_workspace_bytes(int n_cols, int64_t n_rows);
int anv_moments(const anv_column_t* cols, int n_cols, int64_t n_rows, anv_moments_t* out,
                void* workspace, size_t workspace_bytes, void* stream);

/* ---- K2: binning + histogram pass (replaces the Python UDF bucket_label,
 *      transformers.py:248-280, and the groupBy counts of drift_detector.py:252-264)
 * counts [dev] n_cols * count_stride uint64: slot 0 = nulls, slot b = rows in bin b.
 * The library zeroes `counts` on the stream before accumulating.
 * specs [dev] n_cols; cuts [dev] 8-byte threshold slots. count_stride >= max n_bins+1. */
int anv_hist(const anv_column_t* cols, const anv_binspec_t* specs, const void* cuts, int n_cols,
             int64_t n_rows, uint64_t* counts, int count_stride, void* stream);

/* ---- K1+K2 fused: moments AND histogram in ONE read of the frame (the target frame of
 *      drift_detector.statistics, whose cutoffs come from the source model,
 *      drift_detector.py:229-237). */
int anv_moments_hist(const anv_column_t* cols, const anv_binspec_t* specs, const void* cuts, int n_cols,
                     int64_t n_rows, anv_moments_t* out, uint64_t* counts, int count_stride,
                     void* workspace, size_t workspace_bytes, void* stream);

/* ---- bin-id materialisation (attribute_binning's returned frame, transformers.py:273-280)
 * out_bins [dev] int32: column c is written at out_bins + c * out_stride (elements,
 * out_stride >= n_rows and a multiple of 4); null rows get 0.  max_bins >= every n_bins. */
int anv_bin_assign(const anv_column_t* cols, const anv_binspec_t* specs, const void* cuts, int n_cols,
                   int64_t n_rows, int max_bins, int32_t* out_bins, int64_t out_stride, void* stream);

/* ---- categorical code histogram (groupBy(col).count() on dictionary codes:
 *      stats_generator.py:386-401 mode, :611 countDistinct, drift_detector.py:252-264)
 * cols must be ANV_I32 codes in [0, cardinality); counts slot 0 = nulls, slot 1+code. */
int anv_hist_codes(const anv_column_t* cols, const int32_t* cardinality, int n_cols, int64_t n_rows,
                   uint64_t* counts, int count_stride, void* stream);

/* ---- K3: drift reduce (drift_detector.py:266-335) from source/target counts.
 * counts layout as produced by anv_hist / anv_hist_codes.  kind[c]: 0 = binned numeric
 * (null group joins as key -1), 1 = categorical (null groups never join: one
 * (1e-4,1e-4) row per side that has nulls).  n_slots [dev] per column = n_bins + 1.
 * src_is_p != 0: src_p [dev] holds proportions read from a saved model (:245-250). */
int anv_drift_reduce(const uint64_t* src_counts, const uint64_t* tgt_counts, const double* src_p,
                     int src_is_p, const int32_t* n_slots, const int32_t* kind, int n_cols,
                     int count_stride, int64_t n_src, int64_t n_tgt, anv_drift_t* out, void* stream);

/* ---- K4: exact multi-rank selection (Spark summary() percentiles / approxQuantile,
 *      stats_generator.py:488,813,908; transformers.py:215) by radix select on the
 *      order-preserving integer image of the values (NaN sorts last, -0.0 == 0.0).
 * ranks [dev] n_cols * n_ranks 1-based ranks among the NON-NULL values (0 = skip,
 * n_ranks <= 16); out [dev] n_cols * n_ranks doubles (NaN when skipped).
 * key_bits: 32 when every column is F32/I32 (3 passes), else 64 (7 passes). */
size_t anv_select_workspace_bytes(int n_cols, int n_ranks);
int anv_select_ranks(const anv_column_t* cols, int n_cols, int64_t n_rows, const int64_t* ranks,
                     int n_ranks, int key_bits, double* out, void* workspace, size_t workspace_bytes,
                     void* stream);
/* The same selection, one radix pass at a time, for frames whose ROWS are partitioned (row chunks
 * streamed through one GPU, or row slabs on several GPUs - SURVEY.md 8(e) "row-sharded variant":
 * "quantile select needs one all-reduce per refinement round"):
 *   anv_select_begin                       zero the histograms in the workspace
 *   for pass in 0 .. anv_select_passes(key_bits)-1:
 *     anv_select_accumulate(partition)     once per row partition: adds its digit histogram
 *     [all-reduce(sum) the uint64 region anv_select_hist_region reports, across ranks]
 *     anv_select_advance                   locate every rank's digit; the last pass writes `out`
 * anv_select_ranks is exactly this sequence on one partition. */
int anv_select_passes(int key_bits);
int anv_select_begin(int n_cols, int n_ranks, void* workspace, size_t workspace_bytes, void* stream);
int anv_select_hist_region(int n_cols, int n_ranks, int pass, size_t* offset, size_t* bytes);
int anv_select_accumulate(const anv_column_t* cols, int n_cols, int64_t n_rows, int n_ranks,
                          int key_bits, int pass, void* workspace, size_t workspace_bytes, void* stream);
int anv_select_advance(const anv_column_t* cols, int n_cols, const int64_t* ranks, int n_ranks,
                       int key_bits, int pass, double* out, void* workspace, size_t workspace_bytes,
                       void* stream);

/* ---- K6: HyperLogLog++ registers of approx_count_distinct(col, rsd) (stats_generator.py:
 *      605-608): Spark's XXH64 (seed 42) per-type encoding - I32 hashInt, I64 hashLong,
 *      F32 hashInt(floatToIntBits), F64 hashLong(doubleToLongBits), -0.0 -> 0.0 - then
 *      idx = top p bits, rho = clz(rest)+1, register = max.  regs [dev] (n_cols << p) uint32. */
int anv_hll_registers(const anv_column_t* cols, int n_cols, int64_t n_rows, int p, uint32_t* regs,
                      void* stream);
/* Host helper: the same XXH64 over n UTF-8 strings (Arrow offsets) for the dictionaries of
 * string columns.  bytes/offsets/out are HOST pointers. */
int anv_xxh64_utf8(const uint8_t* bytes, const int64_t* offsets, int64_t n, uint64_t* out);

/* Host helper for partitions LARGER than Spark's 50 000-value head buffer (QuantileSummaries.insert flushes the buffer every
 * head_size insertions and compresses at >= compress_threshold samples; the final compress() inserts the rest): the caller
 * sorts every batch of head_size consecutive non-null values on the device (anv_mode_distinct with all ranks requested) and
 * passes them concatenated, each batch ascending.  Strictly sequential merge / compress, ~2 steps per value.  HOST pointers.
 * Returns the number of samples written to (out_value, out_g, out_delta), or a negative anv_status. */
long long anv_gk_partition_sketch(const double* sorted_batches, long long n_values, long long head_size, double eps,
                                  long long compress_threshold, double* out_value, long long* out_g, long long* out_delta,
                                  long long capacity);

/* ---- exact mode / distinct count of numeric columns (mode_computation's per-column
 *      groupBy+sort jobs, stats_generator.py:386-401; countDistinct, :611): batched LSD
 *      radix sort of the non-null values' order-preserving keys + run-length summary.
 * key_bits 32 (all columns F32/I32) or 64.  Outputs [dev] n_cols each: mode_value (NaN when
 * the column has no non-null value; ties -> smallest value), mode_rows, n_distinct
 * (-0.0 == 0.0, all NaNs equal).  Since the keys end up fully sorted, exact order statistics
 * are free: ranks [dev] n_cols * n_ranks 1-based ranks among the non-null values (0 = skip,
 * n_ranks may be 0) -> rank_values [dev] n_cols * n_ranks (the summary() percentiles of
 * stats_generator.py:488,813,908 without a separate selection pass).
 * mode_value of an ANV_I64 column is NOT a double: its 8-byte slot holds the mode as an int64, bit for bit, and the
 * caller reads it as int64_t (a double is exact only up to 2^53, and Spark returns the mode of a bigint column as a
 * long).  The slot of an empty ANV_I64 column is unspecified (mode_rows 0 tells).  Every other dtype gets a double.
 * rank_values stay doubles for every dtype, like Spark's summary() percentiles of a bigint column. */
size_t anv_mode_distinct_workspace_bytes(int n_cols, int64_t n_rows, int key_bits);
int anv_mode_distinct(const anv_column_t* cols, int n_cols, int64_t n_rows, int key_bits,
                      double* mode_value, int64_t* mode_rows, int64_t* n_distinct, const int64_t* ranks,
                      int n_ranks, double* rank_values, void* workspace, size_t workspace_bytes, void* stream);

/* anv_mode_distinct + the HyperLogLog++ registers of the same columns as a by-product (hll_regs [dev] (n_cols << hll_p)
 * uint32, 4 <= hll_p <= 12; NULL = off): the registers are a max over the SET of values, so the run-summary kernel hashes ONE
 * key per run of the sorted keys instead of a separate pass hashing every value (anv_hll_registers; stats_generator.py:
 * 605-608 next to :386-401).  Registers are identical to anv_hll_registers'. */
int anv_mode_distinct_hll(const anv_column_t* cols, int n_cols, int64_t n_rows, int key_bits, double* mode_value,
                          int64_t* mode_rows, int64_t* n_distinct, const int64_t* ranks, int n_ranks, double* rank_values,
                          int hll_p, uint32_t* hll_regs, void* workspace, size_t workspace_bytes, void* stream);

/* The same results - and, with hll_regs, the same HLL++ registers bit for bit - for F32 / I32 columns WITHOUT sorting
 * them (sort.cu, "two-level bucket count"): sample -> fine splitters (every 32nd also a coarse one) -> the pack step groups
 * every tile's keys by coarse group (one read of the raw column) -> one CTA per chunk of <= 4096 keys of a group moves them
 * into fine-bucket order (keys equal to a splitter - zeros, heavy hitters, discrete values - are only counted) -> one CTA per
 * group counts each fine bucket in a shared-memory hash table sized from its exact count, hashes its distinct keys into
 * the HLL++ registers and selects the requested ranks that land in it.  About 4 words of HBM traffic per key instead of
 * ~14; sizes are exact at every level, so nothing overflows.  n_ranks <= 16; 4 <= hll_p <= 12 (hll_regs NULL = off).
 * The per-column workspace is no larger than anv_mode_distinct's for 32-bit keys from 65 536 rows up. */
size_t anv_mode_distinct_partition_workspace_bytes(int n_cols, int64_t n_rows);
int anv_mode_distinct_partition_hll(const anv_column_t* cols, int n_cols, int64_t n_rows, double* mode_value,
                                    int64_t* mode_rows, int64_t* n_distinct, const int64_t* ranks, int n_ranks,
                                    double* rank_values, int hll_p, uint32_t* hll_regs, void* workspace,
                                    size_t workspace_bytes, void* stream);
/* anv_mode_distinct_partition_hll without the registers. */
int anv_mode_distinct_partition(const anv_column_t* cols, int n_cols, int64_t n_rows, double* mode_value,
                                int64_t* mode_rows, int64_t* n_distinct, const int64_t* ranks, int n_ranks,
                                double* rank_values, void* workspace, size_t workspace_bytes, void* stream);

/* ---- row null counts (nullRows_detection, quality_checker.py:248-272: a UDF counting None over the row's columns,
 *      then groupBy(null_cols_count).count()).  validity [dev] n_bitmaps device pointers to the Arrow bitmaps of the
 *      columns that HAVE one (a column without a bitmap adds nothing; n_cols counts every column and sizes `counts`).
 *      NaN is not null.  counts [dev] n_cols + 1 uint64: slot k = rows with k null columns (zeroed by the library).
 *      keep [dev] ceil(n_rows/32) bitmap words or NULL: bit set where the row's count <= max_keep (max_keep < 0: none).
 *      n_cols <= 131071 (17 bit planes per row count; the grid runs over rows only, so ANV_MAX_LAUNCH_COLS does not apply). */
int anv_row_null_counts(const uint32_t* const* validity, int n_bitmaps, int n_cols, int64_t n_rows, int max_keep,
                        uint64_t* counts, uint32_t* keep, void* stream);

/* ---- exact distinct rows (duplicate_detection, quality_checker.py:122-133: idf.groupby(list_of_cols).count()).
 *      Rows are equal when every column is: null == null (the data under a null lane is ignored), every NaN equals
 *      every NaN, -0.0 == 0.0, otherwise equal bits; string columns compare by dictionary code (the caller maps a
 *      repeated dictionary string to one code).  Hash of each row -> LSD sort of (hash prefix, row) -> every row is
 *      compared with its group's first row, so the result never depends on the hash being unique.
 *      hash_bits caps the hash bits kept in the sort key (0 = all that fit above the row index; 1-8 send nearly every
 *      row through the comparison path, for testing).  n_distinct [dev] 1 int64; first [dev] ceil(n_rows/32) bitmap
 *      words, bit set on the first occurrence of every distinct row (row order).  n_rows >= 2^32 or
 *      n_cols > ANV_MAX_LAUNCH_COLS: ANV_ERR_UNSUPPORTED (rows are compared whole, so a caller cannot split the columns). */
size_t anv_row_distinct_workspace_bytes(int64_t n_rows);
int anv_row_distinct(const anv_column_t* cols, int n_cols, int64_t n_rows, int hash_bits, int64_t* n_distinct,
                     uint32_t* first, void* workspace, size_t workspace_bytes, void* stream);

/* ---- mean / median / mode imputation (imputation_MMM, data_transformer/transformers.py:1369-1676; the MMM treatment of
 *      nullColumns_detection, data_analyzer/quality_checker.py:491-519).
 * anv_impute_fill: one streaming pass per column writes a DENSE output column (no bitmap) of spec.out_dtype:
 *   out[r] = (row r non-null && !(NAN_MISSING && isnan(x[r]))) ? convert(x[r]) : fill.
 * (input dtype -> out_dtype) pairs: F32->F32, F64->F64, I32->I32 (numbers or dictionary codes), I64->I64, I32->F64 and
 * I64->F64 (convert = (double)x); other pairs leave the output unwritten.  ANV_IMPUTE_NAN_MISSING (F32 / F64 inputs): NaN
 * counts as missing, as in Spark's Imputer.  ANV_IMPUTE_ROUND_DOUBLE (I64 -> I64): convert = (long)(double)x, the round trip
 * of Spark's recast to double and back (saturating like Java's d2l; for I32 the identity).  `fill` holds the fill value's
 * bits in the output type (low 4 bytes for 4-byte types): the caller converts the surrogate.
 * specs [dev] n_cols; out_ptrs [dev] n_cols device pointers, each 16-byte aligned with room for n_rows rounded up to a
 * multiple of 4 elements. */
#define ANV_IMPUTE_NAN_MISSING 1
#define ANV_IMPUTE_ROUND_DOUBLE 2
typedef struct {
  int32_t out_dtype; /* anv_dtype of the output column */
  int32_t flags;     /* ANV_IMPUTE_* */
  uint64_t fill;     /* fill value bits in out_dtype */
} anv_impute_spec_t;
int anv_impute_fill(const anv_column_t* cols, const anv_impute_spec_t* specs, void* const* out_ptrs, int n_cols, int64_t n_rows,
                    void* stream);
/* The Imputer's statistics skip NaN as well as null: for every column, out_validity [dev] n_cols * ceil(n_rows/32) words
 * (column c at out_validity + c * ceil(n_rows/32)) gets bit r set where row r is non-null and not NaN (bits past n_rows are
 * 0), and n_nan [dev] n_cols int64 the number of non-null NaN rows (zeroed by the library).  Integer columns: the validity. */
int anv_valid_not_nan(const anv_column_t* cols, int n_cols, int64_t n_rows, uint32_t* out_validity, int64_t* n_nan,
                      void* stream);

/* ---- Spark's Bernoulli row sampler (the DEFAULT path of drift_detector.statistics: use_sampling=True ->
 *      data_sampling.py:122-149 `idf.sample(False, fraction, seed)` / `stat.sampleBy("merge", fractions, seed)`,
 *      drift_detector.py:187-211).  One partition per call: Spark seeds XORShiftRandom with seed + partitionIndex,
 *      draws one nextDouble() per row and keeps the row when x < fraction[stratum].  thresholds [dev] n_strata
 *      uint64 = ceil(fraction * 2^53) (x is a 53-bit integer * 2^-53, so the comparison is exact in integers);
 *      strata [dev] int32 stratum id per row or NULL (every row uses thresholds[0]; ids outside [0, n_strata) are
 *      never kept); keep [dev] ceil(n_rows/32) bitmap words, LSB first.  The stream is generated in parallel by
 *      jumping the GF(2)-linear recurrence ahead (sample.cu). */
uint64_t anv_spark_hash_seed(int64_t seed); /* XORShiftRandom.hashSeed: the generator state after setSeed(seed) */
int anv_spark_sample_mask(int64_t n_rows, int64_t seed, const int32_t* strata, const uint64_t* thresholds,
                          int n_strata, uint32_t* keep, void* stream);

/* ---- synthetic column generator used by bench.py / tests (SURVEY.md 8d): Philox4x32-10
 *      keyed by (seed, column), counter = row.  family: 0 normal(a,b) 1 lognormal(0,b)
 *      2 uniform(a,b) 3 zero-inflated exponential(scale b, 70% zeros).
 *      null_rate in [0,1): validity words written when validity != NULL. */
int anv_synth_f32(float* data, uint32_t* validity, int64_t n_rows, uint64_t seed, uint32_t column,
                  int family, float a, float b, float null_rate, void* stream);
int anv_synth_codes(int32_t* data, uint32_t* validity, int64_t n_rows, uint64_t seed, uint32_t column,
                    int cardinality, float zipf_s, float null_rate, void* stream);
/* The same generators for the row chunk [row0, row0 + n_rows) of a larger frame (row0 % 32 == 0):
 * the chunk is bit-identical to those rows of the whole frame, so streamed / row-sharded runs
 * see the same data as a resident one. */
int anv_synth_f32_rows(float* data, uint32_t* validity, int64_t n_rows, int64_t row0, uint64_t seed,
                       uint32_t column, int family, float a, float b, float null_rate, void* stream);
int anv_synth_codes_rows(int32_t* data, uint32_t* validity, int64_t n_rows, int64_t row0, uint64_t seed,
                         uint32_t column, int cardinality, float zipf_s, float null_rate, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ANOVOS_B200_H */
