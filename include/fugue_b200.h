/* fugue_b200 - C ABI of the H100-native (sm_90a) hot path of a Fugue ExecutionEngine.
 *
 * The reference (fugue-project/fugue v0.9.4) is pure Python and has no FFI of
 * its own; its drop-in boundary is a set of Python ABCs
 * (fugue/execution/execution_engine.py: MapEngine :277-335, SQLEngine :183-274,
 * ExecutionEngine :338-1241).  This header is the C boundary that sits directly
 * below the Python classes in fugue_b200/ that implement those ABCs; every entry
 * point cites the reference code whose arithmetic it replaces.
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on error; the message of the
 *     last error of the calling thread is returned by fb_last_error().
 *   - `dev` is a CUDA device ordinal, `stream` a cudaStream_t (NULL = default
 *     stream).  Calls are asynchronous with respect to the host unless stated.
 *   - all data pointers are DEVICE pointers unless the name ends in `_host`.
 *   - a table is a set of equal-length, fixed-width columns (Arrow primitive
 *     layout: one contiguous little-endian buffer per column, width 1/2/4/8
 *     bytes).  NULLs are carried as a byte-per-row mask column (1 = valid);
 *     fb_bits_to_bytes / fb_bytes_to_bits convert from/to Arrow validity bitmaps.
 *   - no global mutable state; scratch memory is supplied by the caller
 *     (fb_*_scratch_bytes says how much) so nothing is allocated in a timed region.
 */
#ifndef FUGUE_B200_H
#define FUGUE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FB_ABI_VERSION 1
#define FB_MAX_KEYS 8        /* key columns of a PartitionSpec / join / group-by */
#define FB_MAX_COLS 64       /* payload columns moved by one partition call */
#define FB_MAX_PARTITIONS 1024 /* physical partitions handled by one radix pass */

int fb_abi_version(void);
const char* fb_last_error(void);

/* Device discovery: number of SMs and bytes of HBM of device `dev`. */
int fb_device_info(int dev, int* sm_count, size_t* total_mem, int* cc_major, int* cc_minor);

/* ---------------------------------------------------------------------------
 * K1  key tuple -> physical partition id
 * Replaces: fugue_dask/_utils.py:146-169 (_add_hash_index)
 *             pd.util.hash_pandas_object(df[cols], index=False).mod(num)
 *           (same expression in fugue_ray/_utils/dataframe.py:115-118).
 * Bit-exact with pandas for fixed-width key columns; a NULL key cell hashes as
 * the float64 NaN bit pattern (see oracle/hash_partition.py).
 * key_valid[k] may be NULL (column has no NULLs) and key_valid itself may be NULL.
 * --------------------------------------------------------------------------- */
int fb_partition_ids(int dev, void* stream, int64_t nrows, int nkeys,
                     const void* const* key_ptrs, const int32_t* key_widths,
                     const uint8_t* const* key_valid, uint32_t num_partitions,
                     uint32_t* out_pids);

/* The 64-bit row hash itself (before `% num`): used to join / group on key tuples wider than
 * 8 bytes (hash as surrogate key, equality verified afterwards). */
int fb_row_hash64(int dev, void* stream, int64_t nrows, int nkeys, const void* const* key_ptrs,
                  const int32_t* key_widths, const uint8_t* const* key_valid, uint64_t* out_hash);

/* Host-side evaluation of the device's division-free `hash % num` (for tests). */
uint32_t fb_debug_fastmod_host(uint64_t hash, uint32_t num_partitions);

/* ---------------------------------------------------------------------------
 * K1+K2+K3  hash partition of a columnar table  (the map_dataframe hot path)
 * Replaces: PandasMapEngine.map_dataframe's grouping step
 *             fugue/execution/native_execution_engine.py:166-168
 *           and the distributed engines' physical repartition
 *             fugue_dask/execution_engine.py:160-181, 263-303  (hash_repartition)
 *             fugue_dask/_utils.py:44-59, 124-130
 * Output: every column reordered so that rows of physical partition p occupy
 * [part_offsets[p], part_offsets[p+1]); input order is kept inside a partition
 * (stable), so results are deterministic.
 *
 * fb_partition_plan  : pass 1 (histogram) + scan; fills part_offsets (device,
 *                      num_partitions+1 int64) and the plan held in `scratch`.
 * fb_partition_apply : pass 2 (scatter) for any subset of columns, using the
 *                      plan; may be called several times (e.g. column by column
 *                      while later columns are still arriving over PCIe).
 * fb_partition_cols  : plan + apply in one call.
 * --------------------------------------------------------------------------- */
size_t fb_partition_scratch_bytes(int dev, int64_t nrows, uint32_t num_partitions);

int fb_partition_plan(int dev, void* stream, int64_t nrows, int nkeys,
                      const void* const* key_ptrs, const int32_t* key_widths,
                      const uint8_t* const* key_valid, uint32_t num_partitions,
                      void* scratch, size_t scratch_bytes, int64_t* out_part_offsets);

int fb_partition_apply(int dev, void* stream, int64_t nrows, int nkeys,
                       const void* const* key_ptrs, const int32_t* key_widths,
                       const uint8_t* const* key_valid, uint32_t num_partitions,
                       const void* scratch, size_t scratch_bytes,
                       const int64_t* part_offsets, int ncols,
                       const void* const* col_ptrs, const int32_t* col_widths,
                       void* const* out_col_ptrs);

/* fb_partition_apply with tuning arguments (0 = default for each).  `sm_reserve` SMs left free: the fast scatter kernel is persistent and a
 * CTA owns its SM's whole register file, so a kernel that must run at the same time (the multi-GPU
 * barrier / pull kernels of the exchange that overlaps the next column group) needs SMs of its own.
 * `cols_per_launch` is the number of 8-byte columns per group of the fast kernel (default 2).  All groups
 * run side by side in one launch, one group per CTA; when fewer than one SM per group is left free, each
 * group gets a launch of its own.  The name is kept for ABI compatibility. */
int fb_partition_apply_ex(int dev, void* stream, int64_t nrows, int nkeys,
                          const void* const* key_ptrs, const int32_t* key_widths,
                          const uint8_t* const* key_valid, uint32_t num_partitions,
                          const void* scratch, size_t scratch_bytes,
                          const int64_t* part_offsets, int ncols,
                          const void* const* col_ptrs, const int32_t* col_widths,
                          void* const* out_col_ptrs, int sm_reserve,
                          int cols_per_launch /* 8-byte columns per group of the fast kernel, 1..8 */);

/* K4  fused map epilogue: fb_partition_apply whose output column c is not a copy of col_ptrs[c] but
 *   mode 1 (float64): (a * x + b * y) + c    mode 2 (int64): a * x + b * y + c (wrapping)    mode 0: x
 * with x = col_ptrs[c][row], y = maps[c].src2[row] (src2 NULL: no y), evaluated by the movers of the
 * scatter kernel between the gather from the staged tile and the store - the per-partition map of
 * PandasMapEngine.map_dataframe (fugue/execution/native_execution_engine.py:156-164) for maps that
 * are column expressions, with no second pass over the table.  float64 operations are rounded one by
 * one (same result as the expression evaluator K8).  All columns 8 bytes wide and 16-byte aligned,
 * num_partitions <= 256.  a / b / c are the constants' bit patterns.  tail_tmp: device scratch of
 * fb_partition_map_tail_bytes(ncols) bytes (the partial last tile is mapped there first). */
typedef struct {
  const void* src2;
  int32_t mode;
  int32_t reserved;
  uint64_t a, b, c;
} fb_map_unit;
size_t fb_partition_map_tail_bytes(int ncols);
int fb_partition_apply_map(int dev, void* stream, int64_t nrows, int nkeys,
                           const void* const* key_ptrs, const int32_t* key_widths,
                           const uint8_t* const* key_valid, uint32_t num_partitions,
                           const void* scratch, size_t scratch_bytes,
                           const int64_t* part_offsets, int ncols,
                           const void* const* col_ptrs, void* const* out_col_ptrs,
                           const fb_map_unit* maps, void* tail_tmp, int sm_reserve);

int fb_partition_cols(int dev, void* stream, int64_t nrows, int ncols,
                      const void* const* col_ptrs, const int32_t* col_widths,
                      const int32_t* key_col_idx, int nkeys,
                      const uint8_t* const* key_valid, uint32_t num_partitions,
                      void* const* out_col_ptrs, int64_t* out_part_offsets,
                      void* scratch, size_t scratch_bytes);

/* ---------------------------------------------------------------------------
 * One stable pass of an LSD radix sort: rows are reordered by the 8-bit digit
 * (sort_key >> shift) & 255 of an 8-byte UNSIGNED sort key column, keeping the current order
 * inside a digit (same kernels as the hash partition; d_offsets: 257 int64).  Eight passes sort
 * by a 64-bit key; the host layer builds order-preserving keys for ints / doubles / NULLS FIRST|LAST
 * / DESC and sorts (key, row index) pairs, then gathers the payload once (fb_gather_rows).
 * Replaces: pdf.sort_values(presort_keys, ascending=...) fugue/execution/native_execution_engine.py:
 * 107-115, 157-160 (presort) and :350-384 (take).
 * --------------------------------------------------------------------------- */
int fb_radix_pass(int dev, void* stream, int64_t nrows, const void* sort_key_u64, int shift, int ncols,
                  const void* const* col_ptrs, const int32_t* col_widths, void* const* out_col_ptrs,
                  void* scratch, size_t scratch_bytes, int64_t* d_offsets);

/* Arrow validity bitmap (LSB first) <-> byte mask. `bit_offset` is the Arrow
 * array offset. */
int fb_bits_to_bytes(int dev, void* stream, const uint8_t* bits, int64_t bit_offset,
                     int64_t nrows, uint8_t* out_bytes);
int fb_bytes_to_bits(int dev, void* stream, const uint8_t* bytes, int64_t nrows,
                     uint8_t* out_bits, int64_t* out_null_count);

/* ---------------------------------------------------------------------------
 * Segment copy / multi-GPU pull exchange (SURVEY.md 8e steps 3-4): for every column c,
 *   out[c][dst_off[s] .. +len[s]) = table[src_table[s]][c][src_off[s] .. +len[s])
 * d_src_cols is a DEVICE array of (ntables x ncols) column pointers laid out [table][col]; with
 * d_src_table == NULL every segment reads table 0.  The tables may be peer-GPU buffers mapped
 * through symmetric memory: the kernel then pulls the runs over NVLink straight into their final
 * place (no NCCL all-to-all, no staging pass).  ALL pointer arguments are DEVICE memory; max_len
 * (host) is the longest segment, used to size the grid.  No reference counterpart: the reference
 * delegates shuffles to Dask/Spark/Ray (fugue_dask/_utils.py:124-130).
 * --------------------------------------------------------------------------- */
int fb_copy_segments(int dev, void* stream, int ncols, const void* const* d_src_cols,
                     void* const* d_dst_cols, const int32_t* d_widths, int nseg,
                     const int32_t* d_src_table, const int64_t* d_src_off, const int64_t* d_dst_off,
                     const int64_t* d_len, int64_t max_len);
/* The exchange on the COPY ENGINES: nruns independent device-to-device copies (local or peer
 * memory mapped into this process) enqueued on `stream`, one cudaMemcpyAsync each.  The multi-GPU
 * repartition issues ONE run per (source rank, column): the partitions a rank owns are contiguous in
 * every source's partitioned table.  Copy engines need no SM, so the transfer over NVLink overlaps
 * the scatter kernel of the next column group.  src / dst / bytes are HOST arrays. */
int fb_copy_runs_dma(int dev, void* stream, int64_t nruns, const void* const* src, void* const* dst,
                     const size_t* bytes);
/* fb_copy_runs_dma with a stream per run (`streams` = HOST array of cudaStream_t): one call enqueues a
 * whole column group of the exchange on the per-peer streams. */
int fb_copy_runs_dma_streams(int dev, int64_t nruns, const void* const* src, void* const* dst,
                             const size_t* bytes, void* const* streams,
                             int prefer_overlap /* 1: cudaMemcpyBatchAsync + cudaMemcpyFlagPreferOverlapWithCompute */);
/* The same runs pulled by a small persistent TMA kernel (`max_ctas` CTAs, one per SM): one thread per
 * CTA keeps ~14 x 16 KB bulk loads (cp.async.bulk) in flight against the peers' memory, four warps
 * drain the stages into the local destination.  nruns <= 64; src / dst / bytes multiples of 8;
 * src / dst / bytes are HOST arrays. */
int fb_pull_runs_tma(int dev, void* stream, int nruns, const void* const* src, void* const* dst,
                     const size_t* bytes, int max_ctas);

/* ---------------------------------------------------------------------------
 * K6  hash group-by with aggregation (single 8-byte key; other key shapes are packed /
 * dictionary-coded into 8 bytes by the host layer)
 * Replaces: ExecutionEngine.aggregate -> SQL -> qpd/pandas groupby
 *             fugue/execution/execution_engine.py:889-939, fugue/column/sql.py:275-334,
 *             fugue/execution/native_execution_engine.py:59-66
 * NULL key forms its own group (fugue_test/execution_suite.py:195-200); NULL values are
 * skipped (SQL semantics), COUNT with a NULL value pointer is COUNT(*).
 *
 * fb_groupby_u64     : clears `table` (fb_groupby_table_bytes) and aggregates nrows rows.
 *                      num_parts > 1 (power of two): the input was hash-partitioned on the key into
 *                      num_parts partitions with fb_partition_cols; keys of partition p then live in
 *                      table region p, so the table is swept region by region (L2-resident atomics).
 *                      d_part_offsets (device, num_parts + 1 row offsets of the partitions, may be
 *                      NULL): the table is then initialised and filled a few regions at a time
 *                      (one launch pair per 32 MB of table), so the regions are still in L2 when
 *                      their atomics arrive.
 *                      d_status[0] != 0 afterwards means the table was too small: retry with
 *                      a larger power-of-two `capacity`.  Value columns are 8 bytes wide.
 * fb_groupby_extract : compacts the groups into out_keys / out_key_valid / out_aggs[a]
 *                      (each 8 bytes per group, capacity + 2 entries allocated by the caller);
 *                      d_status[1] receives the number of groups.  d_out_aggs is a DEVICE array
 *                      of naggs device pointers.  Group order is unspecified.
 *
 * Deviations (the corrected two-pass variance, DESIGN §7i): FB_AGG_DEV_F64 and FB_AGG_DEV2_F64 read
 * the f64 values of their column like FB_AGG_SUM_F64, and each needs, in the same call, an
 * FB_AGG_SUM_F64 with the same value and validity pointers and an FB_AGG_COUNT with the same validity
 * pointer (rejected otherwise).  After the other aggregates of a row's group are complete, the call adds
 * d = x - SUM / COUNT of the row's group into DEV and d * d into DEV2, for every valid x.  With m = COUNT,
 * M2 = sum over the group of (x - mean)^2 = max(0, DEV2 - DEV^2 / m).  A NaN or +-inf value makes DEV
 * and DEV2 NaN.  Several DEV (or DEV2) accumulators of the same column and validity each receive the full sum.
 * fb_segmented_scan and the frame kernels reject both ops.
 *
 * Cross deviations (covariance and regression, DESIGN §7k): an FB_AGG_CODEV_F64 accumulator at index a names
 * x through val_ptrs[a] and the pair validity p through val_valid[a].  Its y is the value column of accumulator
 * a + 1, which must be an FB_AGG_DEV_F64 with the same validity pointer p.  The call must also hold an
 * FB_AGG_SUM_F64 of (x, p), an FB_AGG_SUM_F64 of (y, p) and an FB_AGG_COUNT of p (rejected otherwise).  For every
 * row where p is set, the call adds dx * dy into CODEV, with dx = x - SUM(x) / COUNT and dy = y - SUM(y) / COUNT
 * of the row's group.  With m = COUNT, DEVx and DEVy the deviation sums of x and y over the same rows,
 * Sxy = sum over the group of (x - mean x)(y - mean y) = CODEV - DEVx * DEVy / m.
 *
 * Higher deviations (skewness and kurtosis, DESIGN §7m): FB_AGG_DEV3_F64 and FB_AGG_DEV4_F64 are tied like
 * FB_AGG_DEV2_F64 to an FB_AGG_SUM_F64 of the same value and validity pointers and an FB_AGG_COUNT of the same
 * validity pointer (rejected otherwise), and receive d^3 and d^4 with the same d.  With delta = DEV / m the central
 * sums follow exactly: M2 = DEV2 - m delta^2, M3 = DEV3 - 3 delta DEV2 + 2 m delta^3,
 * M4 = DEV4 - 4 delta DEV3 + 6 delta^2 DEV2 - 3 m delta^4.  A NaN or +-inf value makes them NaN.
 * --------------------------------------------------------------------------- */
#define FB_MAX_AGGS 16
enum {
  FB_AGG_SUM_F64 = 0,
  FB_AGG_SUM_I64 = 1,
  FB_AGG_COUNT = 2,
  FB_AGG_MIN_I64 = 3,
  FB_AGG_MAX_I64 = 4,
  FB_AGG_MIN_F64 = 5,
  FB_AGG_MAX_F64 = 6,
  FB_AGG_DEV_F64 = 7,
  FB_AGG_DEV2_F64 = 8,
  FB_AGG_CODEV_F64 = 9,
  FB_AGG_DEV3_F64 = 10,
  FB_AGG_DEV4_F64 = 11
};
size_t fb_groupby_table_bytes(int64_t capacity, int naggs);
int fb_groupby_u64(int dev, void* stream, int64_t nrows, const void* keys, const uint8_t* key_valid,
                   int naggs, const void* const* val_ptrs, const uint8_t* const* val_valid,
                   const int32_t* agg_ops, int64_t capacity, uint32_t num_parts, void* table,
                   int64_t* d_status, const int64_t* d_part_offsets);
int fb_groupby_extract(int dev, void* stream, int64_t capacity, int naggs, const int32_t* agg_ops,
                       const void* table, void* out_keys, uint8_t* out_key_valid,
                       void* const* d_out_aggs, int64_t* d_status);

/* ---------------------------------------------------------------------------
 * K9  segmented inclusive scan (window functions of a ColumnMap over the logical partitions)
 * Replaces: the per-logical-partition pandas call of PandasMapEngine.map_dataframe
 *             fugue/execution/native_execution_engine.py:156-164
 *           for running totals, forward fill, ranks and partition-wide aggregates.
 * Segment s is rows [d_offsets[s], d_offsets[s + 1]) (device, nseg + 1 int64, d_offsets[0] == 0,
 * d_offsets[nseg] == nrows, empty segments allowed).  For every column c and row i the scan restarts at
 * every segment start and writes, over the rows of i's segment up to and including i whose mask byte
 * valid[c] is non-zero (valid[c] NULL: every row):
 *   out_count[c][i]  the number of those rows (int64)
 *   out_vals[c][i]   ops[c] over their 8-byte values vals[c]: FB_AGG_SUM_I64 (wrapping), FB_AGG_SUM_F64,
 *                    FB_AGG_MIN/MAX_I64, FB_AGG_MIN/MAX_F64 (IEEE totalOrder, the input's own bit pattern);
 *                    0 where the count is 0.  FB_AGG_COUNT reads no values (vals[c] may be NULL).
 * out_vals[c] / out_count[c] may be NULL (not written).  Results are bit-identical from run to run
 * (fixed combination order; f64 sums are not in row order).  ops, vals, valid, out_vals and out_count
 * are HOST arrays of ncols <= FB_SCAN_MAX_COLS entries; scratch: fb_segmented_scan_scratch_bytes.
 * --------------------------------------------------------------------------- */
#define FB_SCAN_MAX_COLS 8
size_t fb_segmented_scan_scratch_bytes(int64_t nrows, int ncols);
int fb_segmented_scan(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets, int ncols,
                      const int32_t* ops, const void* const* vals, const uint8_t* const* valid,
                      void* const* out_vals, int64_t* const* out_count, void* scratch, size_t scratch_bytes);

/* K9  segmented moments: over the same segments, per column c and row i, the valid rows of i's segment up to
 * and including i (f64 values vals[c], mask valid[c] or NULL):
 *   out_count[c][i]  their number m (int64)
 *   out_m2[c][i]     M2 = sum of (x - mean)^2 over them (f64), 0 where m = 0; NaN once a NaN or +-inf is among them
 * The state (n, mean, M2) is combined with Chan, Golub & LeVeque's pairwise update; a value enters as
 * (1, x, x - x).  Same launch sequence and fixed combination order as fb_segmented_scan: bit-identical runs.
 * vals, valid, out_count and out_m2 are HOST arrays of ncols <= FB_SCAN_MAX_COLS entries (an output may be
 * NULL: not written); scratch: fb_segmented_moments_scratch_bytes. */
size_t fb_segmented_moments_scratch_bytes(int64_t nrows, int ncols);
int fb_segmented_moments(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets, int ncols,
                         const void* const* vals, const uint8_t* const* valid, int64_t* const* out_count,
                         void* const* out_m2, void* scratch, size_t scratch_bytes);

/* K9  segmented co-moments: over the same segments, per pair c and row i, the rows of i's segment up to and
 * including i where both x and y are valid (f64 values xs[c] / ys[c], masks x_valid[c] / y_valid[c] or NULL,
 * ANDed by the kernel):
 *   out_count[c][i]               their number m (int64)
 *   out_mean_x[c][i], out_mean_y  the means of x and y over them (f64)
 *   out_sxx[c][i], out_syy, out_sxy  Sxx = sum of (x - mean x)^2, Syy likewise, Sxy = sum of (x - mean x)(y - mean y)
 * All f64 outputs are 0 where m = 0.  A NaN or +-inf in x or y of a pair row makes Sxx, Syy and Sxy NaN from that
 * row on; a mean then becomes what the sum of its values over m gives (+-inf, or NaN).  The state (n, mean x,
 * mean y, Sxx, Syy, Sxy) is combined with Chan's pairwise update, whose cross term is dx * dy * na * nb / n; a
 * pair enters as (1, x, y, z, z, z) with z = (x - x) * (y - y).  Same launch sequence and fixed combination order
 * as fb_segmented_scan: bit-identical runs.  Every pointer argument but d_offsets and scratch is a HOST array of
 * npairs <= FB_SCAN_MAX_COLS entries; an output may be NULL (not written); scratch:
 * fb_segmented_comoments_scratch_bytes. */
size_t fb_segmented_comoments_scratch_bytes(int64_t nrows, int npairs);
int fb_segmented_comoments(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets, int npairs,
                           const void* const* xs, const uint8_t* const* x_valid, const void* const* ys,
                           const uint8_t* const* y_valid, int64_t* const* out_count, void* const* out_mean_x,
                           void* const* out_mean_y, void* const* out_sxx, void* const* out_syy,
                           void* const* out_sxy, void* scratch, size_t scratch_bytes);

/* K9  segmented shape moments: over the same segments, per column c and row i, the valid rows of i's segment up to
 * and including i (f64 values vals[c], mask valid[c] or NULL):
 *   out_count[c][i]                 their number m (int64)
 *   out_m2[c][i], out_m3, out_m4    Mk = sum of (x - mean)^k over them (f64), 0 where m = 0; NaN once a NaN or +-inf
 *                                   is among them
 * The state (n, mean, M2, M3, M4) is combined with Pebay's pairwise update; a value enters as (1, x, z, z, z) with
 * z = x - x.  Same launch sequence and fixed combination order as fb_segmented_scan: bit-identical runs.  vals,
 * valid and the outputs are HOST arrays of ncols <= FB_SCAN_MAX_COLS entries (an output may be NULL: not written);
 * scratch: fb_segmented_shape_moments_scratch_bytes. */
size_t fb_segmented_shape_moments_scratch_bytes(int64_t nrows, int ncols);
int fb_segmented_shape_moments(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets, int ncols,
                               const void* const* vals, const uint8_t* const* valid, int64_t* const* out_count,
                               void* const* out_m2, void* const* out_m3, void* const* out_m4, void* scratch,
                               size_t scratch_bytes);

/* K9  segmented exponentially weighted moments (pandas' ewm): over the same segments, per column c and row i, the
 * observations of i's segment up to and including i.  An observation is a row whose f64 value vals[c] is valid
 * (valid[c], or NULL: every row) and not NaN.  Observation j carries the weight w_j beta^(p_last - p_j), p_last being
 * the position of the last of them, beta = 1 - alpha[c]:
 *   positions[c] FB_EWM_ROWS          p = the row index (pandas' ignore_na=False)
 *                FB_EWM_OBSERVATIONS  p = the observation ordinal (ignore_na=True)
 *                FB_EWM_TIMES         p = times[c][i] (int64) times time_scale[c], beta = 1/2: 0.5^(dt / halflife)
 * w = 1 for the segment's first observation and, with adjust[c], for every other; without adjust, observation k
 * weighs alpha T_(k-1), T being the running total weight (T_1 = 1, T_k = T_(k-1) (beta^(p_k - p_(k-1)) + alpha)).
 * Writes
 *   out_count[c][i]                          the number of observations (int64)
 *   out_mean[c][i], out_w, out_w2, out_c     the weighted mean, W = sum of the weights, W2 = sum of their squares and
 *                                            C = sum of w (x - mean)^2 (f64), 0 where the count is 0
 * Without adjust, W, W2 and C are taken with every weight divided by the total (so W = 1 up to rounding): pandas' T
 * overflows or underflows over long partitions with gaps, and mean, C / W and W2 / W^2 do not depend on the scale.
 * A row without an observation repeats the previous row's values.  Once a +-inf is among the observations C is NaN
 * and the mean is what the weighted sum gives (+-inf, or NaN).  Position differences are exact int64 differences.
 * The state (count, first and last position, first value and its weight, W, W2, mean, C of the others) is combined
 * with a decayed, weighted Chan update; same launch sequence and fixed combination order as fb_segmented_scan: bit-identical runs.
 * alpha must be in (0, 1]; time_scale (1 / halflife) finite and > 0 for FB_EWM_TIMES (times and time_scale may be NULL
 * when no column uses times).  Every pointer argument but d_offsets and scratch is a HOST array of
 * ncols <= FB_SCAN_MAX_COLS entries (an output may be NULL: not written); scratch: fb_segmented_ewm_scratch_bytes. */
#define FB_EWM_ROWS 0
#define FB_EWM_OBSERVATIONS 1
#define FB_EWM_TIMES 2
size_t fb_segmented_ewm_scratch_bytes(int64_t nrows, int ncols);
int fb_segmented_ewm(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets, int ncols,
                     const void* const* vals, const uint8_t* const* valid, const double* alpha, const int32_t* adjust,
                     const int32_t* positions, const void* const* times, const double* time_scale,
                     int64_t* const* out_count, void* const* out_mean, void* const* out_w, void* const* out_w2,
                     void* const* out_c, void* scratch, size_t scratch_bytes);

/* K9  moving-window aggregate: ROWS BETWEEN start AND end over the same segments.  For row i of segment
 * [a, b) the frame is rows [max(a, i + start), min(b - 1, i + end)] (may be empty); a negative bound is
 * PRECEDING, 0 CURRENT ROW, a positive one FOLLOWING.  FB_FRAME_UNBOUNDED_START / _END in `flags` make a
 * side unbounded (clip to a / b - 1) and its bound is ignored; any int64 bound is accepted and clipped,
 * start > end with both sides bounded is an error.  Writes, per column and row, the count of valid rows in
 * the frame and ops[c] over them, 0 where the count is 0: the contract of fb_segmented_scan, with every
 * combination in a fixed order (bit-identical runs) and f64 sums made of the frame's own values only.
 * Both bounds given and width end - start + 1 <= FB_FRAME_TILE_MAX_WIDTH: one pass, each CTA stages its
 * rows plus the width - 1 halo in shared memory.  Otherwise: block prefix / suffix scans in scratch and
 * a combine pass.  Scratch: fb_window_frame_scratch_bytes (0 on the one-pass path).
 * --------------------------------------------------------------------------- */
#define FB_FRAME_UNBOUNDED_START 1
#define FB_FRAME_UNBOUNDED_END 2
#define FB_FRAME_TILE_MAX_WIDTH 1024
size_t fb_window_frame_scratch_bytes(int64_t nrows, int ncols, int64_t start, int64_t end, int flags);
int fb_window_frame(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets, int64_t start,
                    int64_t end, int flags, int ncols, const int32_t* ops, const void* const* vals,
                    const uint8_t* const* valid, void* const* out_vals, int64_t* const* out_count, void* scratch,
                    size_t scratch_bytes);

/* K9  value frames: RANGE BETWEEN start AND end over the same segments, as two calls.
 * fb_window_range_bounds writes, per row i, the first and last row d_lo[i] / d_hi[i] of its frame (int64;
 * d_hi[i] < d_lo[i]: empty).  Every segment is sorted by one presort key, NULL keys last: d_keys holds the
 * key as 8-byte values (int64 for FB_RANGE_KEY_I64, uint64 for FB_RANGE_KEY_U64, f64 for FB_RANGE_KEY_F64)
 * and d_key_valid its validity (NULL: all valid; a float key's NaN rows must be cleared in it); -0.0 equals
 * 0.0.  descending != 0: the keys descend.  start / end are the offsets as 8-byte patterns of the key
 * class's type (int64 offsets for both integer classes, f64 offsets for FB_RANGE_KEY_F64).  For a non-NULL
 * key k_i, row j with a non-NULL key k_j is in the frame when k_i + start <= k_j <= k_i + end (descending:
 * k_i - end <= k_j <= k_i - start): exact integer sums (a sum past the type's range selects nothing on
 * that side), one IEEE f64 addition for f64 keys.  A NULL key's frame is its NULL peers.  Either way
 * FB_FRAME_UNBOUNDED_START / _END extend a side to the segment's first / last row.  Cost O(log distance)
 * per row (a galloping search from the row).  Scratch: fb_window_range_bounds_scratch_bytes.
 * fb_window_bounded writes, per column c and row i, the count of valid rows in [d_lo[i], d_hi[i]] clamped
 * to [0, nrows) and ops[c] over them, 0 where the count is 0: the contract of fb_window_frame for any
 * intervals (no monotonicity assumed).  An aligned power-of-two block tree (level l: op and count of rows
 * [m 2^l, (m + 1) 2^l)) answers each interval from at most two blocks per level: O(log width) per row,
 * bit-identical runs, f64 sums made of the frame's own values.  Scratch: fb_window_bounded_scratch_bytes
 * (16 bytes per row and column). */
#define FB_RANGE_KEY_I64 0
#define FB_RANGE_KEY_U64 1
#define FB_RANGE_KEY_F64 2
size_t fb_window_range_bounds_scratch_bytes(int64_t nseg);
int fb_window_range_bounds(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                           const void* d_keys, const uint8_t* d_key_valid, int key_class, int descending,
                           uint64_t start, uint64_t end, int flags, int64_t* d_lo, int64_t* d_hi, void* scratch,
                           size_t scratch_bytes);
size_t fb_window_bounded_scratch_bytes(int64_t nrows, int ncols);
int fb_window_bounded(int dev, void* stream, int64_t nrows, const int64_t* d_lo, const int64_t* d_hi, int ncols,
                      const int32_t* ops, const void* const* vals, const uint8_t* const* valid, void* const* out_vals,
                      int64_t* const* out_count, void* scratch, size_t scratch_bytes);
/* fb_window_tree builds only the tree of fb_window_bounded, for kernels that walk it (fb_range_join_count /
 * _emit).  Scratch (fb_window_bounded_scratch_bytes(nrows, ncols) bytes) receives, with T the node count of
 * levels >= 1 (the sum of nrows >> l for l >= 1) and off[l] the sum of nrows >> k for 1 <= k < l: the 8-byte
 * value of column c's node m of level l at word c T + off[l] + m, then its int64 count at word ncols T +
 * c T + off[l] + m.  Node (l, m) covers rows [m 2^l, (m + 1) 2^l) and exists for m < nrows >> l; level 0 is
 * the input itself.  Same ops, validity rules and fixed combination order as fb_window_bounded. */
int fb_window_tree(int dev, void* stream, int64_t nrows, int ncols, const int32_t* ops, const void* const* vals,
                   const uint8_t* const* valid, void* scratch, size_t scratch_bytes);

/* K9  value heads: FIRST_VALUE / LAST_VALUE / NTH_VALUE over a frame, NULLs respected.  Row i's frame [lo, hi] is
 * either its ROWS frame (d_lo == d_hi == NULL: segments d_offsets, start / end / flags exactly as fb_window_frame,
 * found by the same arithmetic) or [d_lo[i], d_hi[i]] clamped to [0, nrows) (both given, as fb_window_range_bounds
 * writes them; d_offsets unused).  For each of the ncols <= FB_SCAN_MAX_COLS columns c the picked row is
 * lo + nths[c] - 1 (nths[c] >= 1) or hi (nths[c] == FB_VALUE_LAST); an empty frame, a pick past hi or a NULL at the
 * picked row (valid[c][j] == 0) gives out_valid[c][i] = 0 and an all-zero value, else out_vals[c][i] is the
 * widths[c]-byte value (1 / 2 / 4 / 8) of vals[c] at the picked row and out_valid[c][i] = 1.  Any nths[c] >= 1 is
 * accepted (one past nrows selects nothing).  One thread per row, one launch for every column: no bound array is
 * written.  nths, widths, vals, valid (NULL, or entries NULL: all valid), out_vals and out_valid (entries required)
 * are HOST arrays. */
#define FB_VALUE_LAST 0
int fb_window_value(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets, int64_t start,
                    int64_t end, int flags, const int64_t* d_lo, const int64_t* d_hi, int ncols, const int64_t* nths,
                    const int32_t* widths, const void* const* vals, const uint8_t* const* valid,
                    void* const* out_vals, uint8_t* const* out_valid);

/* K9  distribution heads over the segments of fb_segmented_scan.  d_heads[i] != 0 marks a row that starts a peer
 * group (rows equal on every ORDER BY key; a segment start always starts one, marked or not).  With N = b - a the
 * row count of row i's segment [a, b) and [pf, pl] its peer group, writes (any output may be NULL):
 *   d_percent_rank[i]  (pf - a) / (N - 1), 0 when N = 1 (f64, one IEEE division of two exact integers)
 *   d_cume_dist[i]     (pl - a + 1) / N (f64, likewise)
 *   d_ntile[c][i]      NTILE(ntiles[c]) (int64, ntiles[c] >= 1): with s = N / n and L = N - n s, rows r = i - a below
 *                      L (s + 1) take bucket 1 + r / (s + 1), the rest 1 + L + (r - L (s + 1)) / s; 1 + r when s = 0
 * for nntile <= FB_SCAN_MAX_COLS NTILE columns (ntiles and d_ntile are HOST arrays).  Three launches: the first
 * and last head row of every tile of 2048 rows, one CTA scanning those into the last head before and first head
 * after every tile, then the rows: O(1) per row for any peer-group size.  Scratch:
 * fb_window_distribution_scratch_bytes. */
size_t fb_window_distribution_scratch_bytes(int64_t nrows);
int fb_window_distribution(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                           const uint8_t* d_heads, double* d_percent_rank, double* d_cume_dist, int nntile,
                           const int64_t* ntiles, int64_t* const* d_ntile, void* scratch, size_t scratch_bytes);

/* ---------------------------------------------------------------------------
 * K10 exact order statistics per segment: PERCENTILE_CONT / PERCENTILE_DISC / MEDIAN of one column over the
 *     segments [d_offsets[s], d_offsets[s + 1]) of fb_segmented_scan (logical partitions, sorted groups)
 * Replaces: a pandas function per logical partition (fugue/execution/native_execution_engine.py:156-164)
 *           for groupby().quantile(q).
 * d_vals holds 8-byte values of value_class (FB_RANGE_KEY_I64 / _U64 / _F64: narrower types widened by the
 * host, strings as dictionary ranks), d_valid their validity (NULL: all valid).  NULL rows and f64 NaN are
 * skipped; the non-NULL values of a segment are ordered ascending, -0.0 equal to 0.0, ties by row.  m is
 * their number, written to d_count[s].  For each of the nq <= FB_QUANTILE_MAX_Q pairs (qs[j] in [0, 1],
 * kinds[j]), outs[j] receives per segment:
 *   FB_QUANTILE_CONT  f64: h = q (m - 1), lo = floor(h), frac = h - lo; x[lo] if frac == 0, else
 *                     x[lo] + (x[lo + 1] - x[lo]) frac, every step one IEEE f64 op (values converted to f64 by
 *                     their class, uint64 as unsigned); 0 where m = 0.
 *   FB_QUANTILE_DISC  int64: the row at sorted position max(ceil(q m) - 1, 0) (q m one f64 multiply); -1
 *                     where m = 0.  The caller gathers the value (fb_gather_rows), for any column type.
 * Segments of at most FB_QUANTILE_TILE_ROWS rows are sorted in shared memory by the CTA whose window of that
 * many rows they start in (the column is read once); longer segments are sorted by fb_radix_pass over their
 * rows only, then picked.  The path depends on the segment length alone and both give the same results.
 * qs, kinds and outs are HOST arrays.  Scratch: fb_quantile_scratch_bytes, where long_rows is the number of
 * rows in segments longer than FB_QUANTILE_TILE_ROWS (an upper bound is fine).  With long segments the call
 * synchronises `stream` twice (their number and their key range decide the radix passes).
 * --------------------------------------------------------------------------- */
#define FB_QUANTILE_MAX_Q 16
#define FB_QUANTILE_TILE_ROWS 2048
#define FB_QUANTILE_CONT 0
#define FB_QUANTILE_DISC 1
size_t fb_quantile_scratch_bytes(int dev, int64_t nrows, int64_t long_rows);
int fb_segmented_quantile(int dev, void* stream, int64_t nrows, int64_t nseg, const int64_t* d_offsets,
                          const void* d_vals, const uint8_t* d_valid, int value_class, int nq, const double* qs,
                          const int32_t* kinds, int64_t* d_count, void* const* outs, void* scratch,
                          size_t scratch_bytes);

/* ---------------------------------------------------------------------------
 * K7  hash equi-join on one 8-byte key (other key shapes are packed by the host layer)
 * Replaces: NativeExecutionEngine.join -> triad PandasUtils.join -> pd.merge
 *             fugue/execution/native_execution_engine.py:230-241
 *           schema rule: fugue/dataframe/utils.py:152-226 (host side)
 * NULL keys never match (fugue_test/execution_suite.py:533-543).
 *
 *   num_parts > 1 (power of two, same value in build and probe): both inputs were hash-partitioned
 *   on the key with fb_partition_cols into num_parts partitions; the table is then used region by
 *   region (one region per partition) and stays L2-resident (radix join).
 *   fb_join_build_u64        multimap of the build side (capacity: power of two > nbuild,
 *                            table: fb_join_table_bytes(capacity)); d_status[0] != 0: overflow;
 *                            d_part_offsets (device, num_parts + 1, may be NULL): clear + fill a
 *                            few regions at a time so that they stay in L2
 *   fb_join_probe_count_u64  matches per probe row (outer != 0: unmatched rows count 1); out_first
 *                            (optional): build row of the first match, -1 if none - handed back to
 *                            fb_join_probe_write_u64 (with the counts) it lets rows with one output
 *                            pair skip the second walk of the table
 *   fb_exclusive_scan_i64    counts -> output offsets (out[n] entries) and the total
 *   fb_join_probe_write_u64  (probe_row, build_row) index pairs; build_row = -1 for the
 *                            NULL-extended row of an outer join
 *   fb_join_mark_matched     matched[build_row] = 1 (right / full outer joins)
 *   fb_gather_rows           dst[c][o] = src[c][idx[o]] (idx < 0 -> NULL): all pointer tables
 *                            and widths are DEVICE arrays
 *   fb_scatter_rows          the inverse: dst[c][idx[i]] = src[c][i] for widths 1 / 2 / 4 / 8, and
 *                            dst_valid[c][idx[i]] = src_valid[c][i] (1 where src_valid[c] is NULL) for
 *                            every column whose dst_valid[c] is not NULL; one thread per row moves all
 *                            columns, so idx is read once.  PRECONDITION: idx is a permutation of
 *                            [0, n) (an argsort result); a repeated or out-of-range entry is a race or an
 *                            out-of-bounds store, and is not checked.  Pointer tables and widths are
 *                            DEVICE arrays; both validity tables must be given (entries may be NULL)
 * --------------------------------------------------------------------------- */
size_t fb_join_table_bytes(int64_t capacity);
int fb_join_build_u64(int dev, void* stream, int64_t nbuild, const void* keys, const uint8_t* key_valid,
                      int64_t capacity, uint32_t num_parts, void* table, int64_t* d_status,
                      const int64_t* d_part_offsets);
int fb_join_probe_count_u64(int dev, void* stream, int64_t nprobe, const void* keys,
                            const uint8_t* key_valid, int64_t capacity, uint32_t num_parts,
                            const void* table, int outer, int64_t* out_counts, int64_t* out_first);
int fb_join_probe_write_u64(int dev, void* stream, int64_t nprobe, const void* keys,
                            const uint8_t* key_valid, int64_t capacity, uint32_t num_parts,
                            const void* table, int outer, const int64_t* offsets, int64_t* out_probe_idx,
                            int64_t* out_build_idx, const int64_t* counts, const int64_t* first);
int fb_join_mark_matched(int dev, void* stream, const int64_t* build_idx, int64_t n, uint8_t* matched);
size_t fb_exclusive_scan_scratch_bytes(int64_t n);
int fb_exclusive_scan_i64(int dev, void* stream, int64_t n, const int64_t* in, int64_t* out,
                          int64_t* out_total, void* scratch, size_t scratch_bytes);
/* Stream compaction: out_idx receives, in increasing order, the row numbers whose mask byte is
 * non-zero (at most n entries); *d_count (device) their number.  Used by semi/anti joins, set
 * operations, dropna, take. */
size_t fb_compact_scratch_bytes(int64_t n);
int fb_compact_indices(int dev, void* stream, const uint8_t* mask, int64_t n, int64_t* out_idx,
                       int64_t* d_count, void* scratch, size_t scratch_bytes);
int fb_gather_rows(int dev, void* stream, int ncols, const void* const* d_src_cols, void* const* d_dst_cols,
                   const int32_t* d_widths, const uint8_t* const* d_src_valid, uint8_t* const* d_dst_valid,
                   const int64_t* idx, int64_t n);
int fb_scatter_rows(int dev, void* stream, int ncols, const void* const* d_src_cols, void* const* d_dst_cols,
                    const int32_t* d_widths, const uint8_t* const* d_src_valid, uint8_t* const* d_dst_valid,
                    const int64_t* idx, int64_t n);

/* As-of join search (B200ExecutionEngine.asof_join; pandas.merge_asof semantics).  The right side is sorted by
 * (key, as-of value); run r is rows [d_run_offsets[r], d_run_offsets[r + 1]) of one key, and d_right_codes holds
 * their as-of values as unsigned 64-bit order codes (sort.py _unsigned_order_key) of key_class FB_RANGE_KEY_*.
 * PRECONDITION: the codes ascend within every run (the host passes argsort_rows results); it is not checked.
 * One thread per left row i: d_run[i] is its run (-1: none), d_left_codes[i] its own code, d_left_valid[i] == 0
 * (NULL allowed) a NULL as-of value, which matches nothing.  The candidate is, in the run:
 *   FB_ASOF_BACKWARD  the last row with code <= the row's (< without allow_exact_matches)
 *   FB_ASOF_FORWARD   the first row with code >= the row's (>)
 *   FB_ASOF_NEAREST   the closer of those two; on equal distance the backward one
 * With has_tolerance, a candidate farther than `tolerance` (an int64 >= 0 in storage units for the integer
 * classes, the bits of an f64 for FB_RANGE_KEY_F64) is no candidate.  Integer distances are exact; a float
 * distance is one f64 subtraction (0 for equal values).  d_out[i] = d_right_rows[candidate] (the row before the
 * sort), -1 where there is none. */
#define FB_ASOF_BACKWARD 0
#define FB_ASOF_FORWARD 1
#define FB_ASOF_NEAREST 2
int fb_asof_search(int dev, void* stream, int64_t nleft, const int64_t* d_run, const int64_t* d_run_offsets,
                   const uint64_t* d_left_codes, const uint8_t* d_left_valid, const uint64_t* d_right_codes,
                   const int64_t* d_right_rows, int key_class, int direction, int allow_exact_matches,
                   int has_tolerance, uint64_t tolerance, int64_t* d_out);

/* Range join (B200ExecutionEngine.range_join): every left row with every interval of its run that holds its
 * value.  The right side holds only intervals that can match (valid key, start and end, start <= end), sorted by
 * (key, start) stably; run r is rows [d_run_offsets[r], d_run_offsets[r + 1]) of one key.  d_start_codes holds
 * their starts as unsigned 64-bit order codes (sort.py _unsigned_order_key), d_end_keys their end codes with the
 * sign bit flipped (code ^ 2^63, read as int64), and d_tree (tree_bytes >= fb_window_bounded_scratch_bytes(nright,
 * 1)) the levels of fb_window_tree with op FB_AGG_MAX_I64 over d_end_keys.  PRECONDITION: the start codes ascend
 * within every run (the host passes argsort_rows results) and the tree was built over these end keys; neither is
 * checked.  One thread per left row i: d_run[i] is its run (-1: none), d_left_codes[i] its value's code of the same
 * class, d_left_valid[i] == 0 (NULL allowed) a NULL value, which matches nothing.  Right row j matches when
 * start_j <= x (< x without FB_RANGE_CLOSED_LEFT in `closed`) and x <= end_j (< end_j without
 * FB_RANGE_CLOSED_RIGHT), compared as unsigned codes.  The rows whose start passes are a prefix [s, p) of the run
 * (one binary search); the hits among them are found from the right, each by a walk over the MAX tree to the
 * next row to the left whose end passes: O(log run + (1 + matches) log run) per left row, whatever the nesting.
 *   fb_range_join_count  d_counts[i] = the matches of row i; outer != 0: an unmatched row counts 1
 *   fb_range_join_emit   with d_offsets the exclusive scan of those counts (fb_exclusive_scan_i64): the pairs
 *                        (d_out_left, d_out_right)[d_offsets[i] + k] = (i, d_right_rows[j_k]) for the row's
 *                        matches j_0 < j_1 < ... in sorted position, i.e. ascending (start, right row); an
 *                        unmatched row of an outer join gets (i, -1) */
#define FB_RANGE_CLOSED_LEFT 1
#define FB_RANGE_CLOSED_RIGHT 2
int fb_range_join_count(int dev, void* stream, int64_t nleft, const int64_t* d_run, const int64_t* d_run_offsets,
                        const uint64_t* d_left_codes, const uint8_t* d_left_valid, int64_t nright,
                        const uint64_t* d_start_codes, const int64_t* d_end_keys, const void* d_tree,
                        size_t tree_bytes, int closed, int outer, int64_t* d_counts);
int fb_range_join_emit(int dev, void* stream, int64_t nleft, const int64_t* d_run, const int64_t* d_run_offsets,
                       const uint64_t* d_left_codes, const uint8_t* d_left_valid, int64_t nright,
                       const uint64_t* d_start_codes, const int64_t* d_end_keys, const void* d_tree,
                       size_t tree_bytes, const int64_t* d_right_rows, int closed, int outer,
                       const int64_t* d_counts, const int64_t* d_offsets, int64_t* d_out_left,
                       int64_t* d_out_right);

/* K7 fast path: inner / left-outer join on one 8-byte key with 4-byte slots (build row + 1; keys are
 * compared through the build key column) and a fused probe -> output assembly.
 *   fb_join2_build  : clear + insert (one 32-bit CAS per build row); d_status[0] = 1 on region overflow,
 *                     d_status[1] = 1 when two build rows share a key (exact)
 *   fb_join2_probe  : pass A - per probe row the match count and the first match (uint32 each), per tile
 *                     of 4096 rows the exclusive output offset (d_tile_base, fb_join2_tiles_bytes() bytes)
 *                     and the output size (*d_total)
 *   fb_join2_emit   : pass B - writes the OUTPUT COLUMNS directly: left columns copied from the probe row,
 *                     right columns gathered from the matched build row (NULL-extended with `outer`; then
 *                     right_valid_dst[c] receives the validity of every right column).  No (probe, build)
 *                     index pairs are materialised, no separate gather pass.
 * Replaces the same reference code as the K7 entry points above (native_execution_engine.py:230-241).
 * left_* / right_* are HOST arrays of device pointers / widths (<= 48 columns per side). */
size_t fb_join2_table_bytes(int64_t capacity);
int fb_join2_build(int dev, void* stream, int64_t nbuild, const void* keys, const uint8_t* key_valid,
                   int64_t capacity, uint32_t num_parts, void* table, int64_t* d_status,
                   const int64_t* d_part_offsets);
size_t fb_join2_tiles_bytes(int64_t nprobe);
int fb_join2_probe(int dev, void* stream, int64_t nprobe, const void* probe_keys, const uint8_t* probe_valid,
                   const void* build_keys, int64_t capacity, uint32_t num_parts, const void* table, int outer,
                   uint32_t* out_cnt, uint32_t* out_first, int64_t* d_tile_base, int64_t* d_total,
                   const int64_t* d_status /* of fb_join2_build: [1] == 0 (no duplicate build keys) lets a
                                              chain end at its first match */);
/* fb_join2_build + fb_join2_probe for hash-partitioned inputs (both sides partitioned on the key into
 * num_parts partitions, offsets on the device): per batch of table regions that fits L2 - clear, insert,
 * probe the probe rows of the same partitions - so that the probe reads a table and build keys that are
 * still L2-resident. */
int fb_join2_build_probe(int dev, void* stream, int64_t nbuild, const void* build_keys, const uint8_t* build_valid,
                         const int64_t* d_build_part_offsets, int64_t nprobe, const void* probe_keys,
                         const uint8_t* probe_valid, const int64_t* d_probe_part_offsets, int64_t capacity,
                         uint32_t num_parts, void* table, int outer, uint32_t* out_cnt, uint32_t* out_first,
                         int64_t* d_tile_base, int64_t* d_total, int64_t* d_status);
int fb_join2_emit(int dev, void* stream, int64_t nprobe, const void* probe_keys, const void* build_keys,
                  int64_t capacity, uint32_t num_parts, const void* table, const uint32_t* cnt,
                  const uint32_t* first, const int64_t* d_tile_base, int nleft, const void* const* left_src,
                  void* const* left_dst, const int32_t* left_widths, int nright, const void* const* right_src,
                  void* const* right_dst, const int32_t* right_widths, const uint8_t* const* right_valid_src,
                  uint8_t* const* right_valid_dst);

/* ---------------------------------------------------------------------------
 * K8  column-expression evaluator (SELECT list / WHERE predicate / assign)
 * Replaces: ExecutionEngine.select / filter / assign -> SQLExpressionGenerator -> SQLEngine.select
 *             fugue/execution/execution_engine.py:736-887, fugue/column/sql.py:275-347,
 *             fugue/execution/native_execution_engine.py:59-66 (qpd on pandas)
 *           expression semantics: fugue/column/expressions.py:219-434; pins
 *             fugue_test/execution_suite.py:85-174 (test_filter / test_select / test_assign)
 *
 * One pass evaluates a whole SELECT list: an accumulator-machine program, compiled on the host, runs
 * over every row.  The accumulator (a row's current value + validity) lives in hardware registers;
 * the second operand of an instruction is a column (read straight from HBM, converted from its
 * storage type), an immediate, or one of FB_EXPR_NREGS temporaries (shared memory, only needed when
 * both sides of an operator are compound).  Values are canonical 64-bit: int64, float64 bits, bool
 * as 0|1.
 *   FB_X_MOV    acc <- B                         FB_X_ST   temp[b] <- acc
 *   FB_X_OUT    output[b] <- acc (converted to out_types[b]; validity to out_valid[b] if non-NULL)
 *   arithmetic / comparisons: acc <- acc op B (FB_X_R*: B op acc), NULL if either side is NULL
 *   FB_X_AND / FB_X_OR: Kleene three-valued logic; FB_X_IS_NULL / FB_X_NOT_NULL / FB_X_COALESCE
 *   flags & FB_XF_B_I2F: convert operand B from int64 to float64 first
 *   FB_X_F2I: truncate toward zero; out of range saturates to INT64_MIN / INT64_MAX; NaN -> INT64_MIN
 *   FB_X_LOOKUP acc <- B[acc]: B (FB_XK_COL, type FB_T_I64 or FB_T_F64) is a per-entry table of imm
 *               8-byte values, not a per-row column; entry acc is read, and the table's validity (if any)
 *               at the same entry.  A NULL accumulator, or an entry number outside [0, imm), gives
 *               NULL and issues no load.  A dictionary-encoded string column is loaded with FB_X_MOV (its
 *               int32 code) and mapped through a per-entry result table (fb_string_like / _length).
 * Scalar functions (CASE / NULLIF / % / numeric functions).  Integer ops are on int64 and wrap; float ops on float64.
 * Rule of these ops only: a NaN result from operands that are not NaN (a domain error) is NULL.
 *   FB_X_SEL     acc <- temp[c] is TRUE ? acc : B, c = flags >> FB_XF_COND_SHIFT, a temporary in [0, FB_EXPR_NREGS)
 *                holding a bool.  A NULL or FALSE condition takes B, with B's validity (CASE WHEN, branch by branch)
 *   FB_X_MOD_I   acc <- acc % B, truncated (sign of acc); B = 0 gives NULL; INT64_MIN % -1 = 0 (FB_X_RMOD_I: B % acc)
 *   FB_X_MOD_F   acc <- fmod(acc, B), exact; B = +-0.0 gives NULL, fmod(+-inf, y) is a domain error (FB_X_RMOD_F)
 *   FB_X_ABS_I   acc <- |acc|, INT64_MIN stays INT64_MIN        FB_X_ABS_F   acc <- fabs(acc) (clears the sign bit)
 *   FB_X_FLOOR_F / FB_X_CEIL_F   IEEE floor / ceil
 *   FB_X_ROUND_F acc <- acc rounded to imm decimal digits (imm in [-18, 18]): imm = 0 is C round (half away from
 *                zero); otherwise round(acc * 10^imm) / 10^imm (imm < 0: round(acc / 10^-imm) * 10^-imm), one IEEE
 *                op per step, and acc itself when the scaled value is +-inf or NaN
 *   FB_X_ROUND_I acc <- acc rounded to a multiple of 10^-imm, half away from zero (imm in [-18, -1]), wrapping
 *   FB_X_SQRT / FB_X_EXP / FB_X_LN / FB_X_LOG10   sqrt (correctly rounded), exp, log, log10 of the float acc
 *   FB_X_POW     acc <- pow(acc, B) (C99 Annex F special cases); FB_X_RPOW: pow(B, acc)
 *   FB_X_GREATEST_I / FB_X_LEAST_I / FB_X_GREATEST_F / FB_X_LEAST_F   the larger / smaller of acc and B; a NULL
 *                side is skipped, so the result is NULL only if both are; floats in IEEE totalOrder
 *                (-NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN), returning that operand's bits
 *   The unary ops among these (ABS, FLOOR, CEIL, ROUND, SQRT, EXP, LN, LOG10) take no operand (FB_XK_NONE).
 * Temporal ops.  A value is an int64 count of a unit (enum fb_time_unit) since 1970-01-01 00:00 UTC; the calendar is
 * the proleptic Gregorian one without leap seconds, every division floors (1969-12-31 23:59:59.5 has second 59), NULL
 * propagates.  Exact for every int64 of FB_TU_NS and FB_TU_US, every int32 of FB_TU_DAY, and for FB_TU_MS / FB_TU_S
 * where the year lies within the range of an int32 day count; elsewhere the result is unspecified, but nothing traps
 * (sums and products wrap, every divisor is a positive constant).
 *   FB_X_MULSAT_I   acc <- acc * B, saturated to INT64_MIN / INT64_MAX; B an immediate >= 1 (rescale to a finer unit)
 *   FB_X_FLOORDIV_I acc <- floor(acc / B); B an immediate >= 1 (rescale to a coarser unit)
 *   FB_X_TS_PART    acc <- field of acc; imm = fb_time_field | fb_time_unit << 8, no operand.  FB_TF_SECOND is the
 *                   whole second 0-59; FB_TF_WEEK / FB_TF_ISOYEAR are those of the week's Thursday (ISO 8601)
 *   FB_X_TS_TRUNC   acc <- acc truncated to the start of its part, in the same unit; imm = fb_time_part | unit << 8
 *   FB_X_TS_INDEX   acc <- whole parts from 1970-01-01 00:00 to acc (weeks: from Monday 1969-12-29); same imm.
 *                   DATEDIFF(part, a, b) is INDEX(b) - INDEX(a)
 *   FB_X_TS_ADDMON  acc <- acc + B calendar months (B of any operand kind, int64): month index y * 12 + m - 1 + B with
 *                   floor arithmetic, the day clamped to the last day of the target month, the time of day kept;
 *                   the unit sits in flags >> FB_XF_UNIT_SHIFT
 * Column types: FB_T_U16 / FB_T_U32 load zero-extended, FB_T_F16 loads its IEEE half value exactly.
 * Stores keep the low bits of an integer (unsigned stores are the signed ones of the same width) and
 * round a float to nearest even (FB_T_F32, FB_T_F16).
 * `program`, the pointer tables and the type arrays are HOST arrays (copied into the launch);
 * column / output pointers are device memory.
 * --------------------------------------------------------------------------- */
#define FB_EXPR_MAX_COLS 16
#define FB_EXPR_MAX_OUTS 16
#define FB_EXPR_MAX_INS 96
#define FB_EXPR_NREGS 4
enum fb_expr_type { FB_T_I8 = 0, FB_T_I16 = 1, FB_T_I32 = 2, FB_T_I64 = 3, FB_T_U8 = 4, FB_T_F32 = 5, FB_T_F64 = 6,
                    FB_T_U16 = 7, FB_T_U32 = 8, FB_T_F16 = 9 };
enum fb_expr_operand { FB_XK_NONE = 0, FB_XK_REG = 1, FB_XK_COL = 2, FB_XK_IMM = 3, FB_XK_NULL = 4 };
#define FB_XF_B_I2F 1
#define FB_XF_COND_SHIFT 8 /* FB_X_SEL: the condition's temporary sits in flags >> 8 */
enum fb_expr_op {
  FB_X_MOV = 0, FB_X_ST = 1, FB_X_OUT = 2,
  FB_X_I2F = 3, FB_X_F2I = 4, FB_X_NEG_I = 5, FB_X_NEG_F = 6, FB_X_NOT = 7, FB_X_IS_NULL = 8,
  FB_X_NOT_NULL = 9, FB_X_TOBOOL_I = 10, FB_X_TOBOOL_F = 11,
  FB_X_ADD_I = 12, FB_X_SUB_I = 13, FB_X_RSUB_I = 14, FB_X_MUL_I = 15,
  FB_X_ADD_F = 16, FB_X_SUB_F = 17, FB_X_RSUB_F = 18, FB_X_MUL_F = 19, FB_X_DIV_F = 20, FB_X_RDIV_F = 21,
  FB_X_LT_I = 22, FB_X_LE_I = 23, FB_X_GT_I = 24, FB_X_GE_I = 25, FB_X_EQ_I = 26, FB_X_NE_I = 27,
  FB_X_LT_F = 28, FB_X_LE_F = 29, FB_X_GT_F = 30, FB_X_GE_F = 31, FB_X_EQ_F = 32, FB_X_NE_F = 33,
  FB_X_AND = 34, FB_X_OR = 35, FB_X_COALESCE = 36, FB_X_RCOALESCE = 37, FB_X_LOOKUP = 38,
  FB_X_SEL = 39, FB_X_MOD_I = 40, FB_X_RMOD_I = 41, FB_X_MOD_F = 42, FB_X_RMOD_F = 43,
  FB_X_ABS_I = 44, FB_X_ABS_F = 45, FB_X_FLOOR_F = 46, FB_X_CEIL_F = 47, FB_X_ROUND_F = 48, FB_X_ROUND_I = 49,
  FB_X_SQRT = 50, FB_X_EXP = 51, FB_X_LN = 52, FB_X_LOG10 = 53, FB_X_POW = 54, FB_X_RPOW = 55,
  FB_X_GREATEST_I = 56, FB_X_LEAST_I = 57, FB_X_GREATEST_F = 58, FB_X_LEAST_F = 59,
  FB_X_MULSAT_I = 60, FB_X_FLOORDIV_I = 61, FB_X_TS_PART = 62, FB_X_TS_TRUNC = 63, FB_X_TS_INDEX = 64,
  FB_X_TS_ADDMON = 65
};
#define FB_EXPR_ROUND_MAX_DIGITS 18
#define FB_XF_UNIT_SHIFT 8 /* FB_X_TS_ADDMON: the unit sits in flags >> 8 (imm is free to hold operand B) */
/* what one count of a temporal value is: date32 = days, date64 = milliseconds, timestamp[s|ms|us|ns] */
enum fb_time_unit { FB_TU_DAY = 0, FB_TU_S = 1, FB_TU_MS = 2, FB_TU_US = 3, FB_TU_NS = 4, FB_TU_COUNT = 5 };
enum fb_time_field {
  FB_TF_YEAR = 0, FB_TF_MONTH = 1, FB_TF_DAY = 2, FB_TF_HOUR = 3, FB_TF_MINUTE = 4, FB_TF_SECOND = 5,
  FB_TF_QUARTER = 6, FB_TF_DOW = 7 /* 0 = Sunday */, FB_TF_ISODOW = 8 /* 1 = Monday ... 7 */, FB_TF_DOY = 9,
  FB_TF_WEEK = 10 /* ISO 8601 */, FB_TF_ISOYEAR = 11, FB_TF_COUNT = 12
};
enum fb_time_part {
  FB_TP_YEAR = 0, FB_TP_QUARTER = 1, FB_TP_MONTH = 2, FB_TP_WEEK = 3 /* starts on Monday */, FB_TP_DAY = 4,
  FB_TP_HOUR = 5, FB_TP_MINUTE = 6, FB_TP_SECOND = 7, FB_TP_COUNT = 8
};
typedef struct fb_expr_ins {
  int32_t op;    /* enum fb_expr_op */
  int32_t kind;  /* enum fb_expr_operand: what operand B is */
  int32_t b;     /* temporary / column / output index */
  int32_t flags; /* FB_XF_* */
  int64_t imm;   /* FB_XK_IMM: the value's raw 64 bits */
} fb_expr_ins;
int fb_eval_expr(int dev, void* stream, int64_t nrows, int ncols, const void* const* col_ptrs,
                 const int32_t* col_types, const uint8_t* const* col_valid, int nins,
                 const fb_expr_ins* program, int nouts, const int32_t* out_types, void* const* out_ptrs,
                 uint8_t* const* out_valid);

/* ---------------------------------------------------------------------------
 * K11 string functions, evaluated once per dictionary entry
 * Replaces: the SQL engine's LIKE and LENGTH on a string column (fugue/column/sql.py:275-347 hands them
 *           to qpd / pandas: Series.str.match / str.len, one Python string per row).
 * A dictionary is the Arrow layout of a string array: entry i is the UTF-8 bytes
 * data[offsets[i], offsets[i + 1]) (offsets: n + 1 int64), valid[i] == 0 marks a NULL entry (valid may be
 * NULL: none).  The results are per entry; K8 maps every row's code to its entry's result (FB_X_LOOKUP).
 *
 * fb_string_length : out[i] = the number of code points of entry i (bytes that are not 10xxxxxx), int64;
 *                    0 for a NULL entry.
 * fb_string_like   : out[i] = 1 when entry i matches the pattern, else 0; out_valid[i] = valid[i] (1 when
 *                    valid is NULL).  NULL entries give 0.  Case-sensitive, whole string.  The host compiles
 *                    the pattern into `tokens` (ntokens <= FB_LIKE_MAX_TOKENS): a literal byte 0..255,
 *                    FB_LIKE_ONE (`_`: exactly one code point) or FB_LIKE_ANY (`%`: any sequence, never two in
 *                    a row).  The FB_LIKE_ANY tokens split the pattern into segments: the first is anchored at
 *                    the start of the string, the last at its end, and each middle segment takes its leftmost
 *                    match after the previous one (correct for LIKE without backtracking).  Matches start on
 *                    code-point boundaries only.  tokens is a HOST array (copied into the launch).
 * One thread per entry, grid-stride; the entries must be valid UTF-8 (Arrow strings are).
 * --------------------------------------------------------------------------- */
#define FB_LIKE_MAX_TOKENS 1024
#define FB_LIKE_ONE 256
#define FB_LIKE_ANY 257
int fb_string_length(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                     const uint8_t* valid, int64_t* out);
int fb_string_like(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                   const uint8_t* valid, int ntokens, const int16_t* tokens, uint8_t* out, uint8_t* out_valid);

/* ---------------------------------------------------------------------------
 * K12 string-building functions, evaluated once per dictionary entry
 * Replaces: the SQL engine's UPPER / LOWER / SUBSTR / TRIM / REPLACE / CONCAT / || on a string column
 *           (one Python string per row in qpd / pandas).
 * Dictionaries have the K11 layout.  A function of one string column is a function of its entry, so the
 * host builds a new dictionary from the old one and maps every row's code through an entry -> new code table
 * (K8: FB_X_MOV, FB_X_LOOKUP).
 *
 * fb_string_transform : one op over n outputs; output i reads entry src[i] (src: DEVICE int64, NULL: entry i).
 *   Measure call (out_data == NULL): out_len[i] = the output's byte length (0 when NULL), out_valid[i] = 1
 *   unless the output is NULL.  Write call: the bytes of output i go to out_data + out_offsets[i] (the host's
 *   exclusive scan of out_len); out_len / out_valid are not read.  A NULL entry gives NULL except in
 *   FB_STR_FORMAT with null_is_empty.  Ops (code points are UTF-8 sequences; other bytes pass unchanged):
 *     FB_STR_COPY    the entry (a gather, with src)
 *     FB_STR_UPPER / FB_STR_LOWER  simple case mapping, one code point to one (fb_casemap.inc, pyarrow's
 *                    utf8_upper / utf8_lower)
 *     FB_STR_SUBSTR  SQLite substr(s, start[, length]) in code points (has_length == 0: no length); start and
 *                    length in [-2^62, 2^62]
 *     FB_STR_LTRIM / FB_STR_RTRIM / FB_STR_TRIM  remove the code points of literal 0 from the start / end / both
 *     FB_STR_REPLACE every non-overlapping match of literal 0, left to right, by literal 1; an empty literal 0
 *                    leaves the entry unchanged
 *     FB_STR_FORMAT  the tokens in order: a literal byte 0..255, or FB_STR_SELF for the entry's bytes.  A NULL
 *                    entry gives NULL (||), or with null_is_empty adds no bytes (CONCAT)
 *   Literals (at most FB_STR_MAX_LITERAL bytes each) and tokens (at most FB_STR_MAX_TOKENS) are HOST arrays,
 *   copied into the launch.
 * fb_string_hash        : out[i] = a 64-bit hash of entry i's bytes, keeping the low `bits` (1..64); 0 for a
 *                         NULL entry.
 * fb_string_first_equal : given the (hash, entry) pairs sorted by unsigned hash, stably (sorted_hash,
 *                         sorted_idx; the entries 0..n-1 before the sort), canon[e] = the smallest entry id
 *                         whose bytes equal entry e's (NULL entries are equal to each other only).  It finds
 *                         the start of e's hash run by binary search and compares forward from there: one
 *                         comparison per entry unless hashes collide.
 * One thread per entry, grid-stride; UPPER / LOWER stage their table (about 12 KB) in shared memory.
 * --------------------------------------------------------------------------- */
#define FB_STR_MAX_LITERAL 256
#define FB_STR_MAX_TOKENS 1024
#define FB_STR_SELF 256
enum fb_str_op {
  FB_STR_COPY = 0, FB_STR_UPPER = 1, FB_STR_LOWER = 2, FB_STR_SUBSTR = 3, FB_STR_LTRIM = 4, FB_STR_RTRIM = 5,
  FB_STR_TRIM = 6, FB_STR_REPLACE = 7, FB_STR_FORMAT = 8
};
int fb_string_transform(int dev, void* stream, int op, int64_t n, const int64_t* offsets, const uint8_t* data,
                        const uint8_t* valid, const int64_t* src, int64_t start, int64_t length, int has_length,
                        int nlit0, const uint8_t* lit0, int nlit1, const uint8_t* lit1, int ntokens,
                        const int16_t* tokens, int null_is_empty, int64_t* out_len, uint8_t* out_valid,
                        const int64_t* out_offsets, uint8_t* out_data);
int fb_string_hash(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                   const uint8_t* valid, int bits, uint64_t* out);
int fb_string_first_equal(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                          const uint8_t* valid, const uint64_t* sorted_hash, const int64_t* sorted_idx,
                          int64_t* canon);

/* ---------------------------------------------------------------------------
 * K13 string casts, evaluated once per dictionary entry
 * Replaces: Arrow's cast(string -> type, safe=False) on the host, which a string column's CAST needed (a copy of
 *           the table to the host and back).
 * Dictionaries have the K11 layout.  Entry i parses to what Arrow's cast(safe=False) of the one string gives
 * (DESIGN.md section 7l):
 *   FB_PARSE_I8 .. FB_PARSE_U64  decimal with an optional '-' (unsigned: none), in the target's range; or 0x / 0X
 *                                and 1 to 2 * bytes hex digits, read as two's complement of the width
 *   FB_PARSE_F32 / FB_PARSE_F64  [+-] digits [. digits] [(e|E) [+-] digits], or [+-] inf / infinity / nan /
 *                                nan(chars) in any case; correctly rounded to the target
 *   FB_PARSE_BOOL                true / false in any case, 1, 0
 *   FB_PARSE_DATE32 / _DATE64    YYYY-MM-DD, a valid day of the proleptic Gregorian calendar
 *   FB_PARSE_TS + unit (FB_TU_S .. FB_TU_NS), + FB_PARSE_TS_ZONED when the target has a time zone:
 *                                YYYY-MM-DD[(T| )HH[:MM[:SS[.f]]]], at most as many fraction digits as the unit
 *                                holds; zoned targets require Z / +-HH / +-HHMM / +-HH:MM after the time and store
 *                                the UTC instant, others refuse an offset; the value must fit int64 in the unit.
 * fb_string_parse : out[i] = the value as one 8-byte word (an integer in the target's storage units; float64
 *                   bits for F64, and the float64 widening of the float32 for F32), out_valid[i] = 1 when it
 *                   parsed, status[i] = FB_PARSE_OK / _NULL (a NULL entry) / _INVALID / _UNDECIDED (a float of
 *                   more than 19 significant digits whose truncation does not decide the rounding).  first_bad
 *                   (one DEVICE uint64) = the smallest i whose status is INVALID or UNDECIDED, or UINT64_MAX.
 * fb_debug_string_parse_host : the same over HOST arrays, on the CPU (no first_bad).
 * One thread per entry, grid-stride.
 * --------------------------------------------------------------------------- */
enum fb_parse_target {
  FB_PARSE_I8 = 0, FB_PARSE_I16 = 1, FB_PARSE_I32 = 2, FB_PARSE_I64 = 3, FB_PARSE_U8 = 4, FB_PARSE_U16 = 5,
  FB_PARSE_U32 = 6, FB_PARSE_U64 = 7, FB_PARSE_F32 = 8, FB_PARSE_F64 = 9, FB_PARSE_BOOL = 10, FB_PARSE_DATE32 = 11,
  FB_PARSE_DATE64 = 12, FB_PARSE_TS = 16, FB_PARSE_TS_ZONED = 8
};
enum fb_parse_status { FB_PARSE_OK = 0, FB_PARSE_NULL = 1, FB_PARSE_INVALID = 2, FB_PARSE_UNDECIDED = 3 };
int fb_string_parse(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                    const uint8_t* valid, int target, uint64_t* out, uint8_t* out_valid, uint8_t* status,
                    uint64_t* first_bad);
int fb_debug_string_parse_host(int64_t n, const int64_t* offsets, const uint8_t* data, const uint8_t* valid,
                               int target, uint64_t* out, uint8_t* out_valid, uint8_t* status);

/* ---------------------------------------------------------------------------
 * K14 casts to string, evaluated once per distinct value
 * Replaces: Python's str() of every distinct value on the host, which a CAST(x AS STRING) needed.
 * Value i is one 8-byte word (values: DEVICE) of a kind; its text is what the host frames write for the cast
 * (DESIGN.md section 7n):
 *   FB_FMT_I64 / FB_FMT_U64   decimal (every integer width, widened)
 *   FB_FMT_BOOL               true / false (any non-zero word is true)
 *   FB_FMT_F64                float64 bits as CPython's repr(): the shortest digits that read back to the value
 *                             (Ryu), fixed notation iff the exponent of the first digit is in [-4, 16), else
 *                             1e+16 / 1.5e-05; nan, inf, -inf, -0.0
 *   FB_FMT_DATE32             days since 1970-01-01 as Arrow's cast: [-]YYYY-MM-DD, years -32767 .. 32767, else
 *                             "<value out of range: n>"
 *   FB_FMT_DATE64             milliseconds: the range holds the floor day, the text is the day truncated toward 0
 *                             (Arrow's cast; n: the milliseconds)
 *   FB_FMT_TS + unit (FB_TU_S .. FB_TU_NS), + FB_FMT_TS_FRAC for the unit's 3 / 6 / 9 fraction digits (not with
 *                             FB_TU_S): Arrow's strftime "%Y-%m-%d %H:%M:%S" of the count, floor semantics before
 *                             1970, with its 32-bit day and 16-bit year arithmetic far from the epoch
 * fb_value_format : measure call (out_data == NULL): out_len[i] = value i's byte length (0 where valid[i] == 0).
 *                   Write call: its bytes go to out_data + out_offsets[i] (the host's exclusive scan of out_len);
 *                   out_len is not read.  valid: DEVICE uint8 per value, or NULL.
 * fb_debug_value_format_host : the same over HOST arrays, on the CPU.
 * One thread per value, grid-stride.
 * --------------------------------------------------------------------------- */
enum fb_format_kind {
  FB_FMT_I64 = 0, FB_FMT_U64 = 1, FB_FMT_BOOL = 2, FB_FMT_F64 = 3, FB_FMT_DATE32 = 4, FB_FMT_DATE64 = 5,
  FB_FMT_TS = 8, FB_FMT_TS_FRAC = 16
};
int fb_value_format(int dev, void* stream, int64_t n, const uint64_t* values, const uint8_t* valid, int kind,
                    int64_t* out_len, const int64_t* out_offsets, uint8_t* out_data);
int fb_debug_value_format_host(int64_t n, const uint64_t* values, const uint8_t* valid, int kind, int64_t* out_len,
                               const int64_t* out_offsets, uint8_t* out_data);

/* ---------------------------------------------------------------------------
 * K15 regular expressions, evaluated once per dictionary entry
 * Replaces: pandas str.contains / str.extract / str.replace(regex=True) and DuckDB's regexp_matches /
 *           regexp_extract / regexp_replace, which ran one Python string per row on the host.
 * Dictionaries have the K11 layout.  The host (fugue_b200/regex.py) compiles a pattern of the RE2 subset into a
 * position automaton: every instruction that consumes a code point is a position (at most FB_REGEX_MAX_STATES).
 * A closure is the list of positions, in leftmost-first priority order, that the empty-width part of the program
 * reaches from one point, with the capture slots set on the way (a bit per slot the call tracks) and the match
 * target FB_REGEX_MAX_STATES.  Closure 2 * r + at_end: row r < FB_REGEX_MAX_STATES follows position r, row
 * FB_REGEX_MAX_STATES starts a match away from the start of the text, row FB_REGEX_MAX_STATES + 1 at its start;
 * at_end = 1 where the point is the end of the text ($ and \z hold only there, ^ and \A only at byte 0).
 *   ascii[b]          positions that accept the ASCII byte b
 *   range_lo / _mask  code points >= 128: range r is [range_lo[r], range_lo[r + 1]) (the last reaches U+10FFFF),
 *                     range_lo[0] == 128, strictly increasing; range_mask[r] the positions that accept it
 *   cl_mask / _accept the closure's positions as a bit set / 1 when it reaches the match
 *   cl_off / ent_*    the closure's entries ent_*[cl_off[c], cl_off[c + 1]) in priority order
 *   restart           1 when a match may start away from the start of the text (a search keeps starting them)
 *   rewrite           REGEXP_REPLACE: a byte 0..255, or FB_REGEX_GROUP + k for the text of slots 2k, 2k + 1
 *   group_pair        REGEXP_EXTRACT: the slot pair k whose text is the result
 * fb_regex_match     : out[i] = 1 when the pattern matches somewhere in entry i (the host anchors a full match
 *                      with \A(?:p)\z), else 0; out_valid[i] = valid[i].  A bit-parallel Thompson machine: the
 *                      live positions are one 64-bit word; per code point it ORs the closures of the live positions
 *                      that accept it and the start closure, and stops at the first accept.
 * fb_regex_transform : the K12 measure / write contract of fb_string_transform (no src).  op FB_REGEX_EXTRACT:
 *                      slot pair group_pair of the leftmost-first match, '' when there is none or it is unset.
 *                      FB_REGEX_REPLACE: the first match replaced by the rewrite; FB_REGEX_REPLACE_ALL: every
 *                      match left to right, where an empty match right after the previous match is skipped
 *                      (RE2's GlobalReplace).  A Pike VM over the same closures: threads in priority order, one per
 *                      position, each with nslots (<= FB_REGEX_MAX_SLOTS) int32 slots; entries of at most 2^31 - 1
 *                      bytes.  A NULL entry gives NULL.
 * fb_debug_regex_host : either call over HOST arrays, on the CPU, by the same per-entry code; for a program of op
 *                      FB_REGEX_MATCH, out_len[i] = the 0 / 1 result and out_valid[i] the validity.
 * prog: a HOST struct (checked); dprog: its bytes on the device.  One thread per entry, grid-stride; the match
 * kernel stages ascii, cl_mask and cl_accept in shared memory.
 * --------------------------------------------------------------------------- */
#define FB_REGEX_MAX_STATES 64
#define FB_REGEX_MAX_RANGES 512
#define FB_REGEX_MAX_CLOSURES (2 * (FB_REGEX_MAX_STATES + 2))
#define FB_REGEX_MAX_ENTRIES (FB_REGEX_MAX_CLOSURES * (FB_REGEX_MAX_STATES + 1))
#define FB_REGEX_MAX_SLOTS 8
#define FB_REGEX_MAX_REWRITE 512
#define FB_REGEX_GROUP 256
enum fb_regex_op { FB_REGEX_MATCH = 0, FB_REGEX_EXTRACT = 1, FB_REGEX_REPLACE = 2, FB_REGEX_REPLACE_ALL = 3 };
typedef struct {
  int32_t npos, nranges, nslots, op;
  int32_t group_pair, nrewrite, restart, reserved;
  uint64_t ascii[128];
  uint64_t range_mask[FB_REGEX_MAX_RANGES];
  uint32_t range_lo[FB_REGEX_MAX_RANGES];
  uint64_t cl_mask[FB_REGEX_MAX_CLOSURES];
  uint8_t cl_accept[FB_REGEX_MAX_CLOSURES];
  uint16_t cl_off[FB_REGEX_MAX_CLOSURES + 1];
  uint8_t ent_target[FB_REGEX_MAX_ENTRIES];
  uint8_t ent_save[FB_REGEX_MAX_ENTRIES];
  int16_t rewrite[FB_REGEX_MAX_REWRITE];
} fb_regex_program;
int fb_regex_match(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                   const uint8_t* valid, const fb_regex_program* prog, const fb_regex_program* dprog, uint8_t* out,
                   uint8_t* out_valid);
int fb_regex_transform(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                       const uint8_t* valid, const fb_regex_program* prog, const fb_regex_program* dprog,
                       int64_t* out_len, uint8_t* out_valid, const int64_t* out_offsets, uint8_t* out_data);
int fb_debug_regex_host(int64_t n, const int64_t* offsets, const uint8_t* data, const uint8_t* valid,
                        const fb_regex_program* prog, int64_t* out_len, uint8_t* out_valid, const int64_t* out_offsets,
                        uint8_t* out_data);

#ifdef __cplusplus
}
#endif
#endif /* FUGUE_B200_H */
