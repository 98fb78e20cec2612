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
 * --------------------------------------------------------------------------- */
#define FB_MAX_AGGS 16
enum {
  FB_AGG_SUM_F64 = 0,
  FB_AGG_SUM_I64 = 1,
  FB_AGG_COUNT = 2,
  FB_AGG_MIN_I64 = 3,
  FB_AGG_MAX_I64 = 4,
  FB_AGG_MIN_F64 = 5,
  FB_AGG_MAX_F64 = 6
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
 * `program`, the pointer tables and the type arrays are HOST arrays (copied into the launch);
 * column / output pointers are device memory.
 * --------------------------------------------------------------------------- */
#define FB_EXPR_MAX_COLS 16
#define FB_EXPR_MAX_OUTS 16
#define FB_EXPR_MAX_INS 96
#define FB_EXPR_NREGS 4
enum fb_expr_type { FB_T_I8 = 0, FB_T_I16 = 1, FB_T_I32 = 2, FB_T_I64 = 3, FB_T_U8 = 4, FB_T_F32 = 5, FB_T_F64 = 6 };
enum fb_expr_operand { FB_XK_NONE = 0, FB_XK_REG = 1, FB_XK_COL = 2, FB_XK_IMM = 3, FB_XK_NULL = 4 };
#define FB_XF_B_I2F 1
enum fb_expr_op {
  FB_X_MOV = 0, FB_X_ST = 1, FB_X_OUT = 2,
  FB_X_I2F = 3, FB_X_F2I = 4, FB_X_NEG_I = 5, FB_X_NEG_F = 6, FB_X_NOT = 7, FB_X_IS_NULL = 8,
  FB_X_NOT_NULL = 9, FB_X_TOBOOL_I = 10, FB_X_TOBOOL_F = 11,
  FB_X_ADD_I = 12, FB_X_SUB_I = 13, FB_X_RSUB_I = 14, FB_X_MUL_I = 15,
  FB_X_ADD_F = 16, FB_X_SUB_F = 17, FB_X_RSUB_F = 18, FB_X_MUL_F = 19, FB_X_DIV_F = 20, FB_X_RDIV_F = 21,
  FB_X_LT_I = 22, FB_X_LE_I = 23, FB_X_GT_I = 24, FB_X_GE_I = 25, FB_X_EQ_I = 26, FB_X_NE_I = 27,
  FB_X_LT_F = 28, FB_X_LE_F = 29, FB_X_GT_F = 30, FB_X_GE_F = 31, FB_X_EQ_F = 32, FB_X_NE_F = 33,
  FB_X_AND = 34, FB_X_OR = 35, FB_X_COALESCE = 36, FB_X_RCOALESCE = 37
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

#ifdef __cplusplus
}
#endif
#endif /* FUGUE_B200_H */
