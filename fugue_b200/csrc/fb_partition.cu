// K1+K2+K3: hash partition of a columnar table on sm_90a.
//
// Replaces the grouping/repartition step of the reference's map path:
//   fugue/execution/native_execution_engine.py:166-168  (safe_groupby_apply)
//   fugue_dask/_utils.py:44-59, 124-130, 146-169        (hash_repartition)
//
// Design (HBM-bound byte movement; no tensor-core work exists on this path):
//   * the row range is cut into contiguous chunks of whole TILE-row tiles (at most
//     2 x #SM of them) plus one tail chunk holding the final partial tile;
//   * pass 1 (fb_rank_tile_kernel for num <= 256, fb_hist_kernel otherwise and for the
//     tail chunk): per-chunk histogram of partition ids (reads the key column(s) only:
//     8 B/row for the benchmark schema); for num <= 256 also one rank record per whole
//     tile (partition id and stable rank of every row, rows per partition), each tile
//     ranked by one warp;
//   * scan  (fb_scan_*_kernel)  : exclusive prefix per partition over chunks, then
//     over partitions -> part_offsets[num+1] and chunk bases;
//   * pass 2, fast path (fb_scatter_tma_kernel; single 8-byte key, 8-byte columns):
//     one persistent CTA per SM = 1 producer warp + 16 consumer warps.  The producer
//     streams (tile, column) units into a ring of 32 KB shared-memory stages with
//     TMA bulk copies (cp.async.bulk + mbarrier complete_tx), running several units
//     ahead of the consumers, across tile and chunk boundaries.  Consumers hash the
//     staged key tile, rank rows stably per partition (ballot match + warp-private
//     counters), build the slot -> source-row map of the partition-ordered tile and
//     then, per column, gather straight from the staged tile and store contiguous
//     runs (one run per partition present in the tile) to global memory.  Running
//     per-partition output cursors live in shared memory for the whole chunk.
//   * pass 2, generic path (fb_scatter_kernel; any widths/keys, partial tiles):
//     register-staged loads, permutation through double-buffered shared memory.
//   Algorithmic traffic 128 B/row (read 64 + write 64) for the 8x8-byte schema;
//   the implementation adds the 8 B/row key re-read of pass 1.
#include <stdlib.h>

#include <mutex>

#include "fb_common.cuh"

namespace {

constexpr int kBlock = 512;             // threads per CTA
constexpr int kItems = 8;               // rows per thread per tile
constexpr int kTile = kBlock * kItems;  // 4096 rows per tile
constexpr int kWarps = kBlock / 32;
constexpr int kCtasPerSm = 2;

struct FbCols {
  const void* src[FB_MAX_COLS];
  void* dst[FB_MAX_COLS];
  int32_t width[FB_MAX_COLS];
  int32_t ncols;
};

struct ChunkGeom {
  int64_t nrows;
  int64_t full_rows;        // rows covered by whole tiles
  int64_t tiles_per_chunk;  // whole tiles per full chunk
  int32_t nchunks_full;     // chunks made of whole tiles
  int32_t nchunks;          // + 1 if there is a partial tail tile
};

inline ChunkGeom make_geom(int dev, int64_t nrows) {
  ChunkGeom g;
  g.nrows = nrows;
  const int64_t ntiles_full = nrows / kTile;
  g.full_rows = ntiles_full * kTile;
  const int64_t max_chunks = (int64_t)fb_sm_count(dev) * kCtasPerSm;
  g.tiles_per_chunk = ntiles_full > 0 ? (ntiles_full + max_chunks - 1) / max_chunks : 1;
  g.nchunks_full = (int32_t)((ntiles_full + g.tiles_per_chunk - 1) / g.tiles_per_chunk);
  g.nchunks = g.nchunks_full + (g.full_rows < nrows ? 1 : 0);
  return g;
}

__host__ __device__ __forceinline__ void chunk_range(const ChunkGeom& g, int c, int64_t& r0, int64_t& r1) {
  if (c < g.nchunks_full) {
    r0 = (int64_t)c * g.tiles_per_chunk * kTile;
    r1 = r0 + g.tiles_per_chunk * kTile;
    if (r1 > g.full_rows) r1 = g.full_rows;
  } else {
    r0 = g.full_rows;
    r1 = g.nrows;
  }
}

template <bool kSingleU64>
__device__ __forceinline__ uint32_t compute_pid(const FbKeys& keys, const FbDiv& dv, int64_t row) {
  uint64_t h;
  if (kSingleU64) {
    h = fb_hash_single_u64(__ldg((const unsigned long long*)keys.ptr[0] + row));
  } else {
    if (keys.digit_shift >= 0)  // one pass of an LSD radix sort on an 8-byte unsigned sort key
      return (uint32_t)(__ldg((const unsigned long long*)keys.ptr[0] + row) >> keys.digit_shift) & (dv.d - 1);
    h = fb_row_hash(keys, row);
  }
  return fb_fastmod(h, dv);
}

// ---------------------------------------------------------------------------
// K1 alone: materialise partition ids (tests, repartition planning)
// ---------------------------------------------------------------------------
template <bool kSingleU64>
__global__ void fb_pid_kernel(FbKeys keys, FbDiv dv, int64_t nrows, uint32_t* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < nrows; i += stride) out[i] = compute_pid<kSingleU64>(keys, dv, i);
}

__global__ void fb_row_hash_kernel(FbKeys keys, int64_t nrows, uint64_t* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < nrows; i += stride) out[i] = fb_row_hash(keys, i);
}

// ---------------------------------------------------------------------------
// Warp-level "which lanes hold my value": kBits ballots instead of the hardware
// MATCH instruction (MATCH.ANY is a slow multi-cycle warp instruction that caps the
// whole kernel; ballots issue at full rate).  `m` starts as the mask of lanes
// that take part.  Bit b is moved to the sign bit so that the ballot's predicate
// and the all-ones / all-zeros select come from one shift each: 5 SASS
// instructions per bit, against 7 for `m &= bit ? bal : ~bal`.
// ---------------------------------------------------------------------------
template <int kBits>
__device__ __forceinline__ unsigned match_lanes(uint32_t v, unsigned m) {
#pragma unroll
  for (int b = 0; b < kBits; ++b) {
    const int s = (int)(v << (31 - b)) >> 31;  // all ones if bit b of v is set, else 0
    const unsigned bal = __ballot_sync(0xFFFFFFFFu, s < 0);
    m &= ~(bal ^ (unsigned)s);
  }
  return m;
}

// ---------------------------------------------------------------------------
// pass 1: per-chunk histogram. hist layout: [chunk][num]
// shared: cnt[kWarps][num] warp-private counters (no atomics)
// ---------------------------------------------------------------------------
constexpr int kHistBlock = 1024;  // 2 CTAs/SM -> full occupancy (32 registers/thread)
constexpr int kHistWarps = kHistBlock / 32;
constexpr int kHistRows = kHistBlock * kItems;

template <bool kSingleU64, int kBits>
__global__ void __launch_bounds__(kHistBlock, 2)
fb_hist_kernel(FbKeys keys, FbDiv dv, uint32_t num, ChunkGeom g, int chunk0, uint32_t* __restrict__ hist) {
  extern __shared__ uint32_t s_cnt[];
  for (uint32_t i = threadIdx.x; i < (uint32_t)kHistWarps * num; i += kHistBlock) s_cnt[i] = 0;
  __syncthreads();
  int64_t row0, row1;
  chunk_range(g, chunk0 + (int)blockIdx.x, row0, row1);
  const unsigned lt = fb_lanemask_lt();
  uint32_t* my = s_cnt + (size_t)(threadIdx.x >> 5) * num;
  for (int64_t base = row0; base < row1; base += kHistRows) {
    uint32_t pid[kItems];
    const bool full = base + kHistRows <= row1;
#pragma unroll
    for (int r = 0; r < kItems; ++r) {
      int64_t row = base + (int64_t)r * kHistBlock + threadIdx.x;
      pid[r] = (full || row < row1) ? compute_pid<kSingleU64>(keys, dv, row) : 0xFFFFFFFFu;
    }
#pragma unroll
    for (int r = 0; r < kItems; ++r) {
      const bool ok = pid[r] != 0xFFFFFFFFu;
      unsigned m = match_lanes<kBits>(pid[r], __ballot_sync(0xFFFFFFFFu, ok));
      if (ok && (m & lt) == 0) my[pid[r]] += (uint32_t)__popc(m);
      __syncwarp();
    }
  }
  __syncthreads();
  uint32_t* out = hist + (size_t)(chunk0 + (int)blockIdx.x) * num;
  for (uint32_t b = threadIdx.x; b < num; b += kHistBlock) {
    uint32_t t = 0;
#pragma unroll 8
    for (int w = 0; w < kHistWarps; ++w) t += s_cnt[(size_t)w * num + b];
    out[b] = t;
  }
}

// ---------------------------------------------------------------------------
// pass 1 for num <= 256 (full tiles): histogram AND the complete ranking of every 4096-row tile, so
// that pass 2 never hashes, matches or counts.  One 12800-byte record per tile in scratch:
//   [0, 4096)       uint8  partition id of every row
//   [4096, 12288)   uint16 rank of the row among the rows of the same partition in this tile
//   [12288, 12800)  uint16 rows per partition in this tile (256 entries)
// Pass 2 loads one record per tile with a single TMA bulk copy.
//
// One warp ranks one whole tile: it walks the rows in order, 32 per round (row t0 + 32 i + lane), and
// keeps 256 uint16 counters of its own in shared memory.  Per round the lanes of one partition find each
// other with ballots, the lowest of them bumps the counter, and every lane's rank is the counter before
// the bump plus the lanes of its partition below it.  The running counter is the exclusive prefix over
// the earlier rows of the tile, so no block-wide prefix and no barrier is needed inside a tile.  The
// tiles of chunk c are dealt to the warps of CTA c; one barrier at the end sums the warps' histograms.
// ---------------------------------------------------------------------------
constexpr int kRankBlock = 512, kRankWarps = kRankBlock / 32;
constexpr int kRankRounds = kTile / 32;  // rounds of 32 rows per tile
constexpr int kRankBatch = 8;            // rounds whose keys are loaded together, one batch ahead
constexpr uint32_t kMetaRank = kTile, kMetaCnt = 3 * kTile, kMetaBytes = 3 * kTile + 512;
static_assert(kRankRounds % kRankBatch == 0, "a tile is a whole number of key batches");

// compute_pid of a row whose 8-byte key is `v` (kStaged shapes: one 8-byte key without validity)
template <bool kSingleU64>
__device__ __forceinline__ uint32_t pid_of_key(const FbKeys& keys, const FbDiv& dv, uint64_t v) {
  if (kSingleU64) return fb_fastmod(fb_hash_single_u64(v), dv);
  return (uint32_t)(v >> keys.digit_shift) & (dv.d - 1);
}

// kStaged (one 8-byte key without validity: hashed, or a radix digit): the keys of the next batch of
// rounds, in this tile or the warp's next one, are loaded into registers while this batch is ranked.
// Other key shapes load in the loop (the loads of a batch are still issued together).
template <bool kSingleU64, int kBits, bool kStaged>
__global__ void __launch_bounds__(kRankBlock, 2)
fb_rank_tile_kernel(FbKeys keys, FbDiv dv, uint32_t num, ChunkGeom g, uint32_t* __restrict__ hist,
                    uint8_t* __restrict__ meta) {
  __shared__ __align__(16) uint16_t s_cnt[kRankWarps * 256];
  __shared__ uint32_t s_hist[256];
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt = fb_lanemask_lt();
  uint16_t* __restrict__ my = s_cnt + warp * 256;
  ((uint4*)my)[lane] = make_uint4(0, 0, 0, 0);
  if (threadIdx.x < 256) s_hist[threadIdx.x] = 0;
  __syncthreads();
  int64_t row0, row1;
  chunk_range(g, (int)blockIdx.x, row0, row1);  // launched over the full chunks only
  constexpr int64_t kStride = (int64_t)kRankWarps * kTile;
  uint32_t acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // rows of partitions 8 lane .. 8 lane + 7 in this warp's tiles
  const unsigned long long* __restrict__ kp = (const unsigned long long*)keys.ptr[0] + lane;
  uint64_t kv[kRankBatch];
  if constexpr (kStaged) {
    if (row0 + (int64_t)warp * kTile < row1) {
#pragma unroll
      for (int b = 0; b < kRankBatch; ++b) kv[b] = __ldg(kp + row0 + (int64_t)warp * kTile + b * 32);
    }
  }
  for (int64_t t0 = row0 + (int64_t)warp * kTile; t0 < row1; t0 += kStride) {
    uint8_t* __restrict__ rec = meta + (size_t)(t0 / kTile) * kMetaBytes;
    uint8_t* __restrict__ rec_id = rec + lane;
    uint16_t* __restrict__ rec_rank = (uint16_t*)(rec + kMetaRank) + lane;
    for (int r0 = 0; r0 < kRankRounds; r0 += kRankBatch) {
      uint32_t pid[kRankBatch];
      if constexpr (kStaged) {
#pragma unroll
        for (int b = 0; b < kRankBatch; ++b) pid[b] = pid_of_key<kSingleU64>(keys, dv, kv[b]);
        // next batch: the rest of this tile, then the first rows of this warp's next tile
        const int64_t nxt = r0 + kRankBatch < kRankRounds ? t0 + (r0 + kRankBatch) * 32 : t0 + kStride;
        if (nxt < row1) {
#pragma unroll
          for (int b = 0; b < kRankBatch; ++b) kv[b] = __ldg(kp + nxt + b * 32);
        }
      } else {
#pragma unroll
        for (int b = 0; b < kRankBatch; ++b)
          pid[b] = compute_pid<kSingleU64>(keys, dv, t0 + (r0 + b) * 32 + (int64_t)lane);
      }
#pragma unroll
      for (int b = 0; b < kRankBatch; ++b) {
        const uint32_t p = pid[b];
        const unsigned m = match_lanes<kBits>(p, 0xFFFFFFFFu);
        const unsigned before = __popc(m & lt);
        const uint32_t old = my[p];
        __syncwarp();  // every lane has read the counter before the lowest lane of its partition bumps it
        if (before == 0) my[p] = (uint16_t)(old + __popc(m));
        __syncwarp();  // the next round reads the bumped counters
        rec_id[(r0 + b) * 32] = (uint8_t)p;
        rec_rank[(r0 + b) * 32] = (uint16_t)(old + before);
      }
    }
    // the counters are the tile's rows per partition: the record's count[256]; then reset them
    const uint4 c = ((const uint4*)my)[lane];
    ((uint4*)(rec + kMetaCnt))[lane] = c;
    acc[0] += c.x & 0xFFFFu; acc[1] += c.x >> 16;
    acc[2] += c.y & 0xFFFFu; acc[3] += c.y >> 16;
    acc[4] += c.z & 0xFFFFu; acc[5] += c.z >> 16;
    acc[6] += c.w & 0xFFFFu; acc[7] += c.w >> 16;
    ((uint4*)my)[lane] = make_uint4(0, 0, 0, 0);
    __syncwarp();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (acc[i] != 0) atomicAdd(&s_hist[lane * 8 + i], acc[i]);
  __syncthreads();
  if (threadIdx.x < num) hist[(size_t)blockIdx.x * num + threadIdx.x] = s_hist[threadIdx.x];
}

// ---------------------------------------------------------------------------
// scan A: one CTA per partition id: exclusive prefix over chunks (in place),
// total -> totals[b].  nchunks <= 2 * SM count (<= 1024 handled generally).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
fb_scan_chunks_kernel(uint32_t* __restrict__ hist, uint32_t num, int32_t nchunks,
                      int64_t* __restrict__ totals) {
  __shared__ uint32_t s_warp[8];
  __shared__ uint32_t s_carry;
  const uint32_t b = blockIdx.x;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int32_t c0 = 0; c0 < nchunks; c0 += 256) {
    int32_t c = c0 + threadIdx.x;
    uint32_t v = c < nchunks ? hist[(size_t)c * num + b] : 0;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
      if (lane >= (unsigned)o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    uint32_t wbase = 0;
    for (unsigned w = 0; w < warp; ++w) wbase += s_warp[w];
    uint32_t carry = s_carry;
    if (c < nchunks) hist[(size_t)c * num + b] = carry + wbase + x - v;
    __syncthreads();
    if (threadIdx.x == 255) s_carry = carry + wbase + x;
    __syncthreads();
  }
  if (threadIdx.x == 0) totals[b] = (int64_t)s_carry;
}

// scan B: single CTA: exclusive prefix over partitions (int64), in place on
// offsets[0..num]; input totals in offsets[0..num-1].
__global__ void __launch_bounds__(1024)
fb_scan_parts_kernel(int64_t* __restrict__ offsets, uint32_t num) {
  __shared__ int64_t s_warp[32];
  __shared__ int64_t s_carry;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (uint32_t b0 = 0; b0 < num; b0 += 1024) {
    uint32_t b = b0 + threadIdx.x;
    int64_t v = b < num ? offsets[b] : 0;
    int64_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int64_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
      if (lane >= (unsigned)o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    int64_t wbase = 0;
    for (unsigned w = 0; w < warp; ++w) wbase += s_warp[w];
    int64_t carry = s_carry;
    if (b < num) offsets[b] = carry + wbase + x - v;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = carry + wbase + x;
    __syncthreads();
  }
  if (threadIdx.x == 0) offsets[num] = s_carry;
}

// ---------------------------------------------------------------------------
// pass 2: scatter.  Dynamic shared memory, addressed from one extern array so
// that every access compiles to LDS/STS with offsets computed once per tile:
//   [0, 2*T*8)                buf[2][T] uint64   column staging, double buffered
//   then uint32 regions (nbp = padded number of bins; bins = num + 1 sentinel that
//   collects the slots past the end of a partial tile):
//     delta[nbp]              (cursor - bin_start) of the current tile, mod 2^32
//     cursor[nbp]             running output row of every partition for this chunk
//     bin_start[nbp]          exclusive prefix of the tile histogram
//     cnt[kWarps][nbp]        warp-private counters -> exclusive prefix over warps
//     scanw[32]               warp totals of the block scan
//   then pid_sorted[T] uint16 partition id of every slot of the permuted tile
// ---------------------------------------------------------------------------
__host__ __device__ inline uint32_t nb_padded(uint32_t num) { return (num + 1 + 3) & ~3u; }

__host__ __device__ inline size_t scatter_smem_bytes(uint32_t num) {
  size_t nbp = nb_padded(num);
  return 2 * (size_t)kTile * 8 + (3 + (size_t)kWarps) * nbp * 4 + 32 * 4 + (size_t)kTile * 2;
}

constexpr int kMaxPer = (FB_MAX_PARTITIONS + 1 + kBlock - 1) / kBlock;  // bins per thread in the scan

struct TileCtx {  // all pointers are into shared memory
  uint64_t* buf;
  uint32_t* delta;
  uint32_t* cursor;
  uint32_t* bin_start;
  uint32_t* cnt;
  uint32_t* scanw;
  uint16_t* pid_sorted;
  uint32_t nbp;
};

template <typename T, bool kFull>
__device__ __forceinline__ void load_col(const void* __restrict__ src, int64_t warp_row0, int warp_rows,
                                         unsigned lane, T (&v)[kItems]) {
  const T* __restrict__ p = (const T*)src + warp_row0 + lane;
#pragma unroll
  for (int r = 0; r < kItems; ++r)
    if (kFull || r * 32 + (int)lane < warp_rows) v[r] = __ldg(p + r * 32);
}

// Moves every column of width sizeof(T): coalesced load -> permute through shared memory ->
// run-coalesced store.  One barrier per column (double buffered staging).
template <typename T, bool kFull>
__device__ __forceinline__ void move_columns(const FbCols& cols, const TileCtx& cx,
                                             const uint32_t (&pos)[kItems], const uint32_t (&dst)[kItems],
                                             int64_t warp_row0, int warp_rows, int tile_rows,
                                             unsigned lane, int& phase) {
  int c = 0;
  while (c < cols.ncols && cols.width[c] != (int)sizeof(T)) ++c;
  if (c >= cols.ncols) return;
  T v[kItems];
  load_col<T, kFull>(cols.src[c], warp_row0, warp_rows, lane, v);
  while (c < cols.ncols) {
    T* __restrict__ buf = (T*)(cx.buf + (size_t)(phase & 1) * kTile);
#pragma unroll
    for (int r = 0; r < kItems; ++r) buf[pos[r]] = v[r];
    int nxt = c + 1;
    while (nxt < cols.ncols && cols.width[nxt] != (int)sizeof(T)) ++nxt;
    if (nxt < cols.ncols) load_col<T, kFull>(cols.src[nxt], warp_row0, warp_rows, lane, v);  // prefetch
    __syncthreads();
    T* __restrict__ out = (T*)cols.dst[c];
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      const int j = k * kBlock + (int)threadIdx.x;
      if (kFull || j < tile_rows) out[dst[k]] = buf[j];
    }
    ++phase;
    c = nxt;
  }
}

template <bool kSingleU64, int kBits, bool kFull, bool kAll8>
__device__ __forceinline__ void scatter_tile(const FbKeys& keys, const FbDiv& dv, const uint32_t num,
                                             const FbCols& cols, const TileCtx& cx,
                                             const int64_t tile_row0, const int tile_rows, int& phase) {
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt = fb_lanemask_lt();
  const uint32_t nb = num + 1;
  const uint32_t nbp = cx.nbp;
  uint32_t* __restrict__ my_cnt = cx.cnt + warp * nbp;
  const int64_t warp_row0 = tile_row0 + (int64_t)warp * (32 * kItems);
  const int warp_rows = tile_rows - (int)warp * (32 * kItems);  // rows of this warp's stripe that exist

  // -- 1. partition ids of my rows (warp-striped: row = warp_row0 + r*32 + lane)
  uint32_t pid[kItems];
#pragma unroll
  for (int r = 0; r < kItems; ++r) {
    const bool ok = kFull || (r * 32 + (int)lane) < warp_rows;
    pid[r] = ok ? compute_pid<kSingleU64>(keys, dv, warp_row0 + r * 32 + lane) : num;
  }

  // -- 2. stable rank inside (warp, partition): ballot match + warp-private counters
  //       (counters are zero here: cleared before the tile loop and at the end of every tile)
  uint32_t pos[kItems];
#pragma unroll
  for (int r = 0; r < kItems; ++r) {
    const unsigned m = match_lanes<kBits + (kFull ? 0 : 1)>(pid[r], 0xFFFFFFFFu);
    const unsigned before = __popc(m & lt);
    uint32_t old = 0;
    if (before == 0) {
      old = my_cnt[pid[r]];
      my_cnt[pid[r]] = old + __popc(m);
    }
    __syncwarp();
    old = __shfl_sync(0xFFFFFFFFu, old, __ffs(m) - 1);
    pos[r] = old + before;
  }
  __syncthreads();

  // -- 3. per partition: exclusive prefix over warps, then block-wide exclusive scan of the
  //       tile histogram.  Thread t owns bins [t*per, t*per + per).
  {
    const uint32_t per = (nb + kBlock - 1) / kBlock;
    const uint32_t b0 = threadIdx.x * per;
    uint32_t tot[kMaxPer];
    uint32_t sum = 0;
#pragma unroll
    for (int i = 0; i < kMaxPer; ++i) {
      tot[i] = 0;
      if ((uint32_t)i < per && b0 + i < nb) {
        uint32_t run = 0;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
          const uint32_t t = cx.cnt[w * nbp + b0 + i];
          cx.cnt[w * nbp + b0 + i] = run;
          run += t;
        }
        tot[i] = run;
        sum += run;
      }
    }
    uint32_t x = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
      if (lane >= (unsigned)o) x += y;
    }
    if (lane == 31) cx.scanw[warp] = x;
    __syncthreads();
    uint32_t run = x - sum;
    {
      const uint32_t wt = lane < kWarps ? cx.scanw[lane] : 0;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) {
        const uint32_t v = __shfl_sync(0xFFFFFFFFu, wt, w);
        if ((unsigned)w < warp) run += v;
      }
    }
#pragma unroll
    for (int i = 0; i < kMaxPer; ++i) {
      if ((uint32_t)i < per && b0 + i < nb) {
        const uint32_t cur = cx.cursor[b0 + i];
        cx.bin_start[b0 + i] = run;
        cx.delta[b0 + i] = cur - run;  // slot j of the permuted tile lands at output row delta + j
        cx.cursor[b0 + i] = cur + tot[i];
        run += tot[i];
      }
    }
  }
  __syncthreads();

  // -- 4. final slot of every row inside the permuted tile; publish the slot -> pid map
#pragma unroll
  for (int r = 0; r < kItems; ++r) {
    pos[r] += cx.bin_start[pid[r]] + my_cnt[pid[r]];
    cx.pid_sorted[pos[r]] = (uint16_t)pid[r];
  }
  __syncthreads();
  // output row of the slots this thread writes (same for every column)
  uint32_t dst[kItems];
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    const int j = k * kBlock + (int)threadIdx.x;
    dst[k] = cx.delta[cx.pid_sorted[j]] + (uint32_t)j;
  }
  // counters are dead from here on: clear them for the next tile (visibility is covered by the
  // barriers of the column loop / the trailing barrier)
  for (uint32_t i = threadIdx.x; i < (uint32_t)kWarps * nbp; i += kBlock) cx.cnt[i] = 0;

  // -- 5. move the columns
  move_columns<uint64_t, kFull>(cols, cx, pos, dst, warp_row0, warp_rows, tile_rows, lane, phase);
  if (!kAll8) {
    move_columns<uint32_t, kFull>(cols, cx, pos, dst, warp_row0, warp_rows, tile_rows, lane, phase);
    move_columns<uint16_t, kFull>(cols, cx, pos, dst, warp_row0, warp_rows, tile_rows, lane, phase);
    move_columns<uint8_t, kFull>(cols, cx, pos, dst, warp_row0, warp_rows, tile_rows, lane, phase);
  }
  __syncthreads();  // staging buffers, delta, pid_sorted are rewritten by the next tile
}

template <bool kSingleU64, int kBits, bool kAll8>
__global__ void __launch_bounds__(kBlock, kCtasPerSm)
fb_scatter_kernel(FbKeys keys, FbDiv dv, uint32_t num, ChunkGeom g, int chunk0,
                  const uint32_t* __restrict__ chunk_base, const int64_t* __restrict__ part_offsets,
                  FbCols cols) {
  extern __shared__ __align__(128) uint64_t smem64[];
  TileCtx cx;
  cx.nbp = nb_padded(num);
  cx.buf = smem64;
  cx.delta = (uint32_t*)(smem64 + 2 * kTile);
  cx.cursor = cx.delta + cx.nbp;
  cx.bin_start = cx.cursor + cx.nbp;
  cx.cnt = cx.bin_start + cx.nbp;
  cx.scanw = cx.cnt + kWarps * cx.nbp;
  cx.pid_sorted = (uint16_t*)(cx.scanw + 32);

  const int chunk = chunk0 + (int)blockIdx.x;
  int64_t chunk_row0, chunk_row1;
  chunk_range(g, chunk, chunk_row0, chunk_row1);

  for (uint32_t b = threadIdx.x; b < cx.nbp; b += kBlock)
    cx.cursor[b] = b < num ? (uint32_t)part_offsets[b] + chunk_base[(size_t)chunk * num + b] : 0u;
  for (uint32_t i = threadIdx.x; i < (uint32_t)kWarps * cx.nbp; i += kBlock) cx.cnt[i] = 0;
  __syncthreads();

  int phase = 0;
  for (int64_t tile_row0 = chunk_row0; tile_row0 < chunk_row1; tile_row0 += kTile) {
    const int64_t left = chunk_row1 - tile_row0;
    if (left >= kTile)
      scatter_tile<kSingleU64, kBits, true, kAll8>(keys, dv, num, cols, cx, tile_row0, kTile, phase);
    else
      scatter_tile<kSingleU64, kBits, false, kAll8>(keys, dv, num, cols, cx, tile_row0, (int)left, phase);
  }
}

// ---------------------------------------------------------------------------
// pass 2, fast path: TMA-pipelined scatter with software write-combining.
//
// A partition-ordered tile written as 8-byte-aligned runs is slow because run
// heads/tails are partial 32-byte sectors (L2 fills them from DRAM and writes them
// back twice); the same traffic with sector-aligned runs comes close to linear stores.  So every
// partition keeps its last (< G) rows per column in a shared-memory carry buffer and
// only whole G-row groups (G * 8 B = one or more full sectors) are stored; the
// carried rows are prepended to the partition's rows of the next tile.  Partial
// stores happen only at chunk heads/tails (2 per partition per column per chunk).
//
// Shared memory (dynamic, one CTA per SM), T = kTile, E = num * (G - 1):
//   ring[S][T] uint64          S x 32 KB stages filled by cp.async.bulk (TMA)
//   carry[ncols + 1][E] uint64 carried rows per column (+1 spare: new carry is written
//                              to the spare buffer, buffers rotate every column step)
//   slotinfo[T + E] uint32     output slot -> (partition << 16 | source descriptor)
//   carryinfo[E] uint16        new carry entry -> source descriptor
//   per-partition uint32 arrays: wpos, kcnt, binfo, bin_start, wstart, wdelta
//   cnt[kWarps][nbp] uint16, scanw[64] uint32, mbarriers
// Source descriptor: [0, T) row of the staged tile; [T, T + E) old carry entry;
// 0xFFFF nothing (phantom row at a chunk head / unused carry entry).
// ---------------------------------------------------------------------------
constexpr int kSwcMaxCols = 8;             // payload columns per launch (carry buffers in smem)
constexpr uint32_t kSwcMaxNum = 256;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Relaxed arrive: releasing a ring stage does not have to order this warp's global stores.
// The stage reads are ordered by issue: the arrive is issued after the instructions that
// consume the LDS results.
__device__ __forceinline__ void mbar_arrive_relaxed(uint32_t bar) {
  asm volatile("mbarrier.arrive.relaxed.cta.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "FB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra FB_DONE;\n"
      "bra FB_WAIT;\n"
      "FB_DONE:\n"
      "}\n" ::"r"(bar), "r"(parity)
      : "memory");
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// 1-D bulk copy global -> shared, completion signalled on an mbarrier (TMA engine; SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar,
                                            uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(bar), "l"(policy)
      : "memory");
}

// ---------------------------------------------------------------------------
// pass 2, fast path v5: warp-specialised scatter (producer / rankers / movers).
//
// In a single-role design, one third of the kernel is the per-tile ranking
// (hash, match, scans), during which no byte moves; the column phase itself runs near the HBM
// peak.  Here the two run concurrently on different warps of the same persistent CTA:
//   warp 24      producer : TMA bulk loads - the rank record of tile t+1 (partition id, rank and
//                           per-partition counts, written by pass 1: nothing is hashed, matched or
//                           counted here and ANY key shape takes this path) and the payload column
//                           tiles of tile t into the ring
//   warps 16-23  rankers  : place tile t+1: advance the write-combining state of every partition,
//                           build the slot list of the tile
//   warps 0-15   movers   : tile t: per column gather from the staged tile / carry, store whole
//                           G-row groups, save the new carry (in place: the per-column barrier
//                           separates the reads of the old carry from the writes of the new one)
// Hand-off through mbarriers: slots_ready (rankers -> movers), slots_free (movers -> rankers, as
// soon as the slot list sits in mover registers), flush_done at chunk ends, full/empty per ring
// stage and per pid buffer.
// Shared memory (one CTA per SM), T = 4096, E = num * (G - 1):
//   ring[S][T] u64 | mbarriers | carry[ncols][E] u64 | slotinfo[T+E] u32 | wpos kcnt binfo
//   wstart wdelta [nbp] u32 | scanw[64] | carryinfo[E] u16 | rank records [2][12800 B]
// ---------------------------------------------------------------------------
constexpr int kWsMoverWarps = 16, kWsRankWarps = 8;
constexpr int kWsMovers = kWsMoverWarps * 32, kWsRankers = kWsRankWarps * 32;
constexpr int kWsThreads = kWsMovers + kWsRankers + 128;  // + producer warpgroup (1 active warp)
// Rows per write-combined group.  16 rows = 128 B = one whole L2 line per store event, so a line never waits
// half-written in L2 for the next tile of its CTA, and DRAM gets it in one write-back.  H100 at 700 W, 100 M rows
// x 8 columns in groups of 2: 5.31 ms at G = 4 (one sector), 5.18 at G = 8, 5.04 at G = 16 (MEASUREMENTS.md).
constexpr int kWsG = 16;
// Groups of other sizes use 4-row (32 B, one sector) groups: a single column per CTA is slower at G = 16, and the
// G = 16 carry (30 KB per column at num = 256) of 3 or more columns leaves fewer than kWsMinStages ring stages.
constexpr int kWsGWide = 4;
constexpr int kWsMinStages = 3;
constexpr int kWsRankItems = 16;  // rows per ranker thread per tile: tile = 256 x 16 = 4096 rows (2048: no faster)
// Registers per thread of each role (setmaxnreg).  The launch gives every thread 65536 / 896 -> 72; the producer
// warpgroup and the rankers hand theirs to the movers, whose G = 16 slot lists (16 slot rounds, 8 carry rounds) do
// not fit 72.  128 x 24 + 256 x 64 + 512 x 88 = 896 x 72.
constexpr uint32_t kWsProducerRegs = 24, kWsRankerRegs = 64, kWsMoverRegs = 88;
static_assert(128 * kWsProducerRegs + kWsRankers * kWsRankerRegs + kWsMovers * kWsMoverRegs <= kWsThreads * 72,
              "setmaxnreg: the roles take more registers than the launch gives the CTA");
// Slot rounds a mover gathers before it stores them: bounds the values live at once (4 and 8 run alike; all 16
// rounds at once spill)
constexpr int kMoveBatch = 8;

// The units of every column group of one launch.  Group k holds units [k * per_group, min(nunits,
// (k + 1) * per_group)).  CTA b moves group b % ngroups over chunks b / ngroups, + S, + 2S, ... with
// S = gridDim.x / ngroups, so the ngroups CTAs of one chunk run side by side on the same tile sequence
// and every rank record is fetched from HBM about once (the siblings find it in L2).
struct WsUnits {
  const uint64_t* src[FB_MAX_COLS];
  uint64_t* dst[FB_MAX_COLS];
  int32_t nunits;
  int32_t per_group;  // <= kSwcMaxCols: carry buffers in shared memory
  int32_t ngroups;
};

// K4, the fused map epilogue: output unit u is not a copy of src[u] but an affine function of one or
// two staged input tiles, computed by the movers right after the gather and before the store:
//   mode 1 (float64): (a * x + b * y) + c, every operation rounded on its own (no FMA contraction), i.e.
//                     exactly what the expression evaluator (K8) gives for `x * a + y * b + c`
//   mode 2 (int64)  : a * x + b * y + c  (wrapping)
// src2 == nullptr: y does not exist (b ignored).  A two-operand unit occupies two ring stages.
struct WsMap {  // indexed like WsUnits
  const uint64_t* src2[FB_MAX_COLS];
  uint64_t a[FB_MAX_COLS], b[FB_MAX_COLS], c[FB_MAX_COLS];
  int32_t mode[FB_MAX_COLS];
};

__device__ __forceinline__ uint64_t ws_apply_map(int mode, bool two, uint64_t x, uint64_t y, uint64_t a, uint64_t b,
                                                 uint64_t c) {
  if (mode == 1) {
    double r = __dmul_rn(__longlong_as_double((long long)a), __longlong_as_double((long long)x));
    if (two) r = __dadd_rn(r, __dmul_rn(__longlong_as_double((long long)b), __longlong_as_double((long long)y)));
    return (uint64_t)__double_as_longlong(__dadd_rn(r, __longlong_as_double((long long)c)));
  }
  if (mode == 2) return a * x + (two ? b * y : 0ULL) + c;
  return x;
}

template <int G, int RI>
__host__ __device__ inline size_t ws_book_bytes(uint32_t num, int ncols) {
  constexpr size_t kT = (size_t)kWsRankers * RI;
  const size_t nbp = nb_padded(num);
  const size_t E = (size_t)num * (G - 1);
  size_t b = 64 * 8;                           // mbarriers
  b += (size_t)ncols * E * 8;                  // carry buffers (in place)
  b += (kT + E) * 4;                           // slotinfo
  b += 5 * nbp * 4 + 64 * 4;                   // per-partition arrays + scanw
  b += ((E * 2 + 15) / 16) * 16;               // carryinfo
  b += 2 * (size_t)kMetaBytes + 128;           // rank records (+ alignment slack)
  return b;
}

__device__ __forceinline__ void mbar_arrive(uint32_t bar) {  // release.cta: publishes prior smem writes
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mover_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kWsMovers) : "memory"); }
__device__ __forceinline__ void ranker_sync() { asm volatile("bar.sync 2, %0;" ::"n"(kWsRankers) : "memory"); }
// warpgroup-wide register reallocation (sm_90a; SASS: USETMAXREG)
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

template <int kBits, int G, int kWsRankItems, bool kMap>
__global__ void __launch_bounds__(kWsThreads, 1)
fb_scatter_ws_kernel(WsUnits units, uint32_t num, ChunkGeom g, int nstages,
                     const uint8_t* __restrict__ meta,
                     const uint32_t* __restrict__ chunk_base, const int64_t* __restrict__ part_offsets,
                     const __grid_constant__ WsMap map) {
  constexpr uint32_t T = (uint32_t)kWsRankers * kWsRankItems;  // rows per tile
  static_assert(T == (uint32_t)kTile, "pass 1 ranks tiles of kTile rows");
  // kcnt keeps the pending count (phantoms included) and the phantom count in 8 bits each
  static_assert(G >= 2 && G <= 16 && (G & (G - 1)) == 0, "G must be a power of two <= 16");
  constexpr uint32_t GM = G - 1;
  constexpr uint32_t kStageBytes = T * 8;
  constexpr int kSlotRounds = ((int)T + (int)kSwcMaxNum * (G - 1) + kWsMovers - 1) / kWsMovers;
  constexpr int kEntryRoundsM = ((int)kSwcMaxNum * (G - 1) + kWsMovers - 1) / kWsMovers;
  extern __shared__ __align__(128) uint64_t smem64[];
  const uint32_t nbp = nb_padded(num);
  const uint32_t E = num * GM;
  // this CTA's column group (units u0 .. u0 + ncols) and chunk sequence (chunk_first, + chunk_step, ...)
  const int grp = (int)blockIdx.x % units.ngroups;
  const int chunk_first = (int)blockIdx.x / units.ngroups, chunk_step = (int)gridDim.x / units.ngroups;
  const int u0 = grp * units.per_group;
  const int ncols = min(units.per_group, units.nunits - u0);
  uint64_t* ring = smem64;
  uint64_t* bars = ring + (size_t)nstages * T;
  uint64_t* carry = bars + 64;
  uint32_t* slotinfo = (uint32_t*)(carry + (size_t)ncols * E);
  uint32_t* wpos = slotinfo + T + E;
  uint32_t* kcnt = wpos + nbp;
  uint32_t* binfo = kcnt + nbp;
  uint32_t* wstart = binfo + nbp;
  uint32_t* wdelta = wstart + nbp;
  uint32_t* scanw = wdelta + nbp;  // [8,16) written per ranker warp, [40] W
  uint16_t* carryinfo = (uint16_t*)(scanw + 64);
  uint8_t* metabuf = (uint8_t*)(((uintptr_t)(carryinfo + E) + 127) & ~(uintptr_t)127);  // TMA dst

  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + 16);
  const uint32_t bar_pid_full = smem_u32(bars + 32), bar_pid_empty = smem_u32(bars + 34);
  const uint32_t bar_slots_ready = smem_u32(bars + 36), bar_slots_free = smem_u32(bars + 37);
  const uint32_t bar_flush_done = smem_u32(bars + 38);

  if (threadIdx.x == 0) {
    for (int s = 0; s < nstages; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, kWsMoverWarps);
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(bar_pid_full + 8 * i, 1);
      mbar_init(bar_pid_empty + 8 * i, kWsRankWarps);
    }
    mbar_init(bar_slots_ready, kWsRankWarps);
    mbar_init(bar_slots_free, kWsMoverWarps);
    mbar_init(bar_flush_done, kWsMoverWarps);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= kWsMoverWarps + kWsRankWarps) {
    // ============================ producer =============================================
    setmaxnreg_dec<kWsProducerRegs>();
    if (warp == kWsMoverWarps + kWsRankWarps && lane == 0) {
      // the payload is read once: evict first.  A rank record is read by every group of its chunk: kept
      // in L2 for the sibling CTAs (H100 at 400 W, 100 M rows x 8 columns in 4 groups: records loaded
      // evict_first 5.94 ms, evict_normal 5.77, evict_last 5.59; MEASUREMENTS.md)
      const uint64_t pol = l2_policy_evict_first(), meta_pol = l2_policy_evict_last();
      const uint32_t ring_s = smem_u32(ring), meta_s = smem_u32(metabuf);
      uint32_t s = 0, ph = 0, seq = 0;
      // pids of the very first tile
      int chunk = chunk_first;
      int64_t r0 = 0, r1 = 0, t0 = 0;
      bool have = chunk < g.nchunks_full;
      if (have) { chunk_range(g, chunk, r0, r1); t0 = r0; }
      auto load_pid = [&](int64_t row0, uint32_t q) {
        const uint32_t b = q & 1, pp = (q >> 1) & 1;
        mbar_wait(bar_pid_empty + 8 * b, pp ^ 1);
        mbar_expect_tx(bar_pid_full + 8 * b, kMetaBytes);
        tma_load_1d(meta_s + b * kMetaBytes, meta + (size_t)(row0 / T) * kMetaBytes, kMetaBytes,
                    bar_pid_full + 8 * b, meta_pol);
      };
      if (have) load_pid(t0, 0);
      while (have) {
        // next tile of this CTA's sequence (for the pid look-ahead)
        int nchunk = chunk;
        int64_t nr0 = r0, nr1 = r1, nt0 = t0 + T;
        bool nhave = true;
        if (nt0 >= r1) {
          nchunk = chunk + chunk_step;
          nhave = nchunk < g.nchunks_full;
          if (nhave) { chunk_range(g, nchunk, nr0, nr1); nt0 = nr0; }
        }
        if (nhave) load_pid(nt0, seq + 1);
        for (int u = u0; u < u0 + ncols; ++u) {
          mbar_wait(bar_empty + 8 * s, ph ^ 1);
          mbar_expect_tx(bar_full + 8 * s, kStageBytes);
          tma_load_1d(ring_s + s * kStageBytes, units.src[u] + t0, kStageBytes, bar_full + 8 * s, pol);
          if (++s == (uint32_t)nstages) { s = 0; ph ^= 1; }
          if constexpr (kMap) {
            if (map.src2[u] != nullptr) {  // second operand of a fused map: the next stage
              mbar_wait(bar_empty + 8 * s, ph ^ 1);
              mbar_expect_tx(bar_full + 8 * s, kStageBytes);
              tma_load_1d(ring_s + s * kStageBytes, map.src2[u] + t0, kStageBytes, bar_full + 8 * s, pol);
              if (++s == (uint32_t)nstages) { s = 0; ph ^= 1; }
            }
          }
        }
        chunk = nchunk; r0 = nr0; r1 = nr1; t0 = nt0; have = nhave;
        ++seq;
      }
    }
    return;
  }

  if (warp >= kWsMoverWarps) {
    // ============================ rankers (8 warps) ====================================
    setmaxnreg_dec<kWsRankerRegs>();
    const unsigned rw = warp - kWsMoverWarps;          // ranker warp 0..7
    const unsigned rtid = threadIdx.x - kWsMovers;     // 0..255
    uint32_t seq = 0, cseq = 0;
    for (int chunk = chunk_first; chunk < g.nchunks_full; chunk += chunk_step, ++cseq) {
      int64_t r0, r1;
      chunk_range(g, chunk, r0, r1);
      if (cseq > 0) mbar_wait(bar_flush_done, (cseq - 1) & 1);  // movers flushed the previous chunk
      ranker_sync();
      for (uint32_t b = rtid; b < nbp; b += kWsRankers) {
        const uint32_t p0 = b < num ? (uint32_t)part_offsets[b] + chunk_base[(size_t)chunk * num + b] : 0u;
        wpos[b] = p0 & ~GM;
        kcnt[b] = (p0 & GM) | ((p0 & GM) << 8);
      }
      ranker_sync();
      for (int64_t t0 = r0; t0 < r1; t0 += T, ++seq) {
        const uint32_t pb = seq & 1, pph = (seq >> 1) & 1;
        mbar_wait(bar_pid_full + 8 * pb, pph);
        const uint8_t* __restrict__ rec = metabuf + pb * kMetaBytes;
        // ---- per partition (thread b < num): tile count, rows to write, new pending state
        const uint32_t b = rtid;
        uint32_t n = 0, w = 0, kold = 0, phold = 0, wp_old = 0;
        if (b < num) n = ((const uint16_t*)(rec + kMetaCnt))[b];
        if (b < num) {
          const uint32_t kc = kcnt[b];
          kold = kc & 0xFFu;
          phold = kc >> 8;
          wp_old = wpos[b];
          const uint32_t end = wp_old + kold + n;
          const uint32_t aend = end & ~GM;
          if (aend > wp_old) {
            w = aend - wp_old;
            wpos[b] = aend;
            kcnt[b] = end - aend;  // phantoms are consumed by the first write
          } else {
            kcnt[b] = (kold + n) | (phold << 8);
          }
          binfo[b] = kold | (w << 8);
        }
        uint32_t xw = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const uint32_t yw = __shfl_up_sync(0xFFFFFFFFu, xw, o);
          if (lane >= (unsigned)o) xw += yw;
        }
        if (lane == 31) scanw[8 + rw] = xw;
        ranker_sync();  // B
        uint32_t bw = xw - w;
        {
          const uint32_t tw = lane < kWsRankWarps ? scanw[8 + lane] : 0;
#pragma unroll
          for (int wi = 0; wi < kWsRankWarps; ++wi) {
            const uint32_t vw = __shfl_sync(0xFFFFFFFFu, tw, wi);
            if ((unsigned)wi < rw) bw += vw;
          }
        }
        // ---- hand-off arrays may be rewritten once the movers hold the previous slot list
        if (seq > 0) mbar_wait(bar_slots_free, (seq - 1) & 1);
        if (b < num) {
          wstart[b] = bw;
          wdelta[b] = wp_old - bw;  // slot j lands at output row wdelta + j
        }
        if (rtid == kWsRankers - 1) scanw[40] = bw + w;  // W: slots to store this tile
        ranker_sync();  // C
        // ---- every new row / old carry entry finds its place.  The rows of this thread (r * 256 + rtid) are read
        //      from the record here, not kept in registers since the top of the tile: the producer fills the
        //      other record buffer meanwhile, and needs this one only for the tile after next.
#pragma unroll
        for (int r = 0; r < kWsRankItems; ++r) {
          const uint32_t row = r * kWsRankers + rtid;
          const uint32_t pb2 = rec[row];
          const uint32_t bi = binfo[pb2];
          const uint32_t i = (bi & 0xFFu) + ((const uint16_t*)(rec + kMetaRank))[row];
          const uint32_t ww = bi >> 8;
          if (i < ww) slotinfo[wstart[pb2] + i] = (pb2 << 16) | row;
          else carryinfo[pb2 * GM + (i - ww)] = (uint16_t)row;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive_relaxed(bar_pid_empty + 8 * pb);  // the record has been read
        if (b < num) {  // the old carry entries of partition b
#pragma unroll
          for (uint32_t i = 0; i < GM; ++i) {
            const uint32_t e = b * GM + i;
            const uint32_t desc = i < phold ? 0xFFFFu : T + e;
            if (i < kold) {
              if (i < w) slotinfo[bw + i] = (b << 16) | desc;
              else carryinfo[e] = (uint16_t)desc;
            }
            if (w + i >= kold + n) carryinfo[e] = 0xFFFFu;
          }
        }
        ranker_sync();  // D: the slot list of this tile is complete
        if (lane == 0) mbar_arrive(bar_slots_ready);
      }
    }
    return;
  }

  // ================================ movers (16 warps) ====================================
  setmaxnreg_inc<kWsMoverRegs>();
  uint32_t s = 0, ph = 0, seq = 0;
  for (int chunk = chunk_first; chunk < g.nchunks_full; chunk += chunk_step) {
    int64_t r0, r1;
    chunk_range(g, chunk, r0, r1);
    for (int64_t t0 = r0; t0 < r1; t0 += T, ++seq) {
      mbar_wait(bar_slots_ready, seq & 1);
      const uint32_t W = scanw[40];
      uint32_t srcd[kSlotRounds], dst[kSlotRounds];
#pragma unroll
      for (int k = 0; k < kSlotRounds; ++k) {
        const uint32_t j = k * kWsMovers + threadIdx.x;
        srcd[k] = 0xFFFFu;
        dst[k] = 0;
        if (j < W) {
          const uint32_t info = slotinfo[j];
          srcd[k] = info & 0xFFFFu;
          dst[k] = wdelta[info >> 16] + j;
        }
      }
      // New carry entries that come from the staged tile.  An entry carried over from an earlier tile keeps
      // its place (its descriptor is T + e: a partition either writes all its pending rows or none), so it
      // is neither read nor rewritten.
      uint32_t csrc[kEntryRoundsM];
#pragma unroll
      for (int q = 0; q < kEntryRoundsM; ++q) {
        const uint32_t e = q * kWsMovers + threadIdx.x;
        const uint32_t d = e < E ? (uint32_t)carryinfo[e] : 0xFFFFu;
        csrc[q] = d < T ? d : 0xFFFFu;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_slots_free);  // the slot list sits in registers now

      for (int u = 0; u < ncols; ++u) {
        mbar_wait(bar_full + 8 * s, ph);
        const uint64_t* __restrict__ st = ring + (size_t)s * T;
        uint64_t* __restrict__ out = units.dst[u0 + u];
        uint64_t* __restrict__ cbuf = carry + (size_t)u * E;
        uint32_t s2 = s;
        bool two = false;
        const uint64_t* __restrict__ st2 = st;
        int mode = 0;
        uint64_t ma = 0, mb = 0, mc = 0;
        if constexpr (kMap) {
          // fused map (K4): rows taken from the staged tile(s) are mapped here; carry entries already are
          // output values
          mode = map.mode[u0 + u];
          two = map.src2[u0 + u] != nullptr;
          if (two) {
            s2 = s + 1 == (uint32_t)nstages ? 0 : s + 1;
            mbar_wait(bar_full + 8 * s2, s2 == 0 ? ph ^ 1 : ph);
            st2 = ring + (size_t)s2 * T;
          }
          ma = map.a[u0 + u]; mb = map.b[u0 + u]; mc = map.c[u0 + u];
        }
        auto staged = [&](uint32_t r) -> uint64_t {
          if constexpr (kMap) return ws_apply_map(mode, two, st[r], st2[r], ma, mb, mc);
          else return st[r];
        };
        // gather from the stage / old carry and store, kMoveBatch slot rounds at a time
#pragma unroll
        for (int k0 = 0; k0 < kSlotRounds; k0 += kMoveBatch) {
          uint64_t v[kMoveBatch];
#pragma unroll
          for (int k = 0; k < kMoveBatch; ++k)
            if (k0 + k < kSlotRounds && srcd[k0 + k] != 0xFFFFu)
              v[k] = srcd[k0 + k] < T ? staged(srcd[k0 + k]) : cbuf[srcd[k0 + k] - T];
#pragma unroll
          for (int k = 0; k < kMoveBatch; ++k)
            if (k0 + k < kSlotRounds && srcd[k0 + k] != 0xFFFFu) out[dst[k0 + k]] = v[k];
        }
        mover_sync();  // every mover has read the old carry of this column: it is overwritten in place
#pragma unroll
        for (int q = 0; q < kEntryRoundsM; ++q)
          if (csrc[q] != 0xFFFFu) cbuf[q * kWsMovers + threadIdx.x] = staged(csrc[q]);
        // all my reads of the stage have completed (their values were consumed by the stores above)
        __syncwarp();
        if (lane == 0) {
          mbar_arrive_relaxed(bar_empty + 8 * s);
          if (kMap && two) mbar_arrive_relaxed(bar_empty + 8 * s2);
        }
        if (++s == (uint32_t)nstages) { s = 0; ph ^= 1; }
        if (kMap && two) {
          if (++s == (uint32_t)nstages) { s = 0; ph ^= 1; }
        }
      }
      // The new carry of column u is read in the next tile after the barrier of column u + 1 of this tile or
      // of column 0 of the next one.  A single column has neither: order it here.
      if (ncols == 1) mover_sync();
    }
    // ---- chunk end: flush the pending rows (partial groups)
    mover_sync();
    for (int u = 0; u < ncols; ++u) {
      uint64_t* __restrict__ out = units.dst[u0 + u];
      const uint64_t* __restrict__ cbuf = carry + (size_t)u * E;
#pragma unroll
      for (int q = 0; q < kEntryRoundsM; ++q) {
        const uint32_t e = q * kWsMovers + threadIdx.x;
        if (e < E) {
          const uint32_t b = e / GM, i = e - b * GM;
          const uint32_t kc = kcnt[b];
          if (i < (kc & 0xFFu) && i >= (kc >> 8)) out[wpos[b] + i] = cbuf[e];
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_flush_done);  // rankers may start the next chunk
  }
}

// ---------------------------------------------------------------------------
// validity bitmap <-> byte mask
// ---------------------------------------------------------------------------
__global__ void fb_bits_to_bytes_kernel(const uint8_t* __restrict__ bits, int64_t bit_offset,
                                        int64_t nrows, uint8_t* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (; i < nrows; i += stride) {
    int64_t j = i + bit_offset;
    out[i] = (bits[j >> 3] >> (j & 7)) & 1;
  }
}

__global__ void fb_bytes_to_bits_kernel(const uint8_t* __restrict__ bytes, int64_t nrows,
                                        uint8_t* __restrict__ out, unsigned long long* null_count) {
  // one thread per output byte
  int64_t nbytes = (nrows + 7) >> 3;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long nulls = 0;
  for (; i < nbytes; i += stride) {
    uint8_t v = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      int64_t r = i * 8 + k;
      if (r < nrows) {
        if (bytes[r]) v |= (uint8_t)(1u << k);
        else ++nulls;
      }
    }
    out[i] = v;
  }
  if (null_count != nullptr && nulls) atomicAdd(null_count, nulls);
}

inline int bits_for(uint32_t num) { return num <= 16 ? 4 : (num <= 256 ? 8 : 10); }

#define FB_DISPATCH_SB(single, bits, LAUNCH)                 \
  do {                                                       \
    if (single) {                                            \
      if (bits == 4) LAUNCH(true, 4);                        \
      else if (bits == 8) LAUNCH(true, 8);                   \
      else LAUNCH(true, 10);                                 \
    } else {                                                 \
      if (bits == 4) LAUNCH(false, 4);                       \
      else if (bits == 8) LAUNCH(false, 8);                  \
      else LAUNCH(false, 10);                                \
    }                                                        \
  } while (0)

template <typename K>
cudaError_t optin(K kernel, size_t bytes) {
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}

// opt in to > 48 KB of dynamic shared memory, once per device
cudaError_t ensure_smem_optin(int dev) {
  static std::mutex mu;
  static uint64_t done = 0;
  std::lock_guard<std::mutex> lock(mu);
  if (dev >= 0 && dev < 64 && (done >> dev) & 1) return cudaSuccess;
  const size_t sc = scatter_smem_bytes(FB_MAX_PARTITIONS);
  const size_t hs = (size_t)kHistWarps * FB_MAX_PARTITIONS * sizeof(uint32_t);
  cudaError_t e = cudaSuccess;
#define FB_OPTIN(S, B)                                                   \
  do {                                                                   \
    if (e == cudaSuccess) e = optin(fb_scatter_kernel<S, B, true>, sc);  \
    if (e == cudaSuccess) e = optin(fb_scatter_kernel<S, B, false>, sc); \
    if (e == cudaSuccess) e = optin(fb_hist_kernel<S, B>, hs);           \
  } while (0)
  {
    int smem_max = 0;
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
#define FB_OPTIN_WS(G)                                                                                        \
  do {                                                                                                        \
    if (e == cudaSuccess) e = optin(fb_scatter_ws_kernel<4, G, kWsRankItems, false>, (size_t)smem_max);       \
    if (e == cudaSuccess) e = optin(fb_scatter_ws_kernel<8, G, kWsRankItems, false>, (size_t)smem_max);       \
    if (e == cudaSuccess) e = optin(fb_scatter_ws_kernel<4, G, kWsRankItems, true>, (size_t)smem_max);        \
    if (e == cudaSuccess) e = optin(fb_scatter_ws_kernel<8, G, kWsRankItems, true>, (size_t)smem_max);        \
  } while (0)
    FB_OPTIN_WS(kWsG);
    FB_OPTIN_WS(kWsGWide);
#undef FB_OPTIN_WS
  }
  FB_OPTIN(true, 4); FB_OPTIN(true, 8); FB_OPTIN(true, 10);
  FB_OPTIN(false, 4); FB_OPTIN(false, 8); FB_OPTIN(false, 10);
#undef FB_OPTIN
  if (e == cudaSuccess && dev >= 0 && dev < 64) done |= (1ull << dev);
  return e;
}

bool single_u64_key(int nkeys, const int32_t* widths, const uint8_t* const* valid) {
  return nkeys == 1 && widths[0] == 8 && (valid == nullptr || valid[0] == nullptr);
}

int fill_keys(FbKeys& k, int nkeys, const void* const* ptrs, const int32_t* widths,
              const uint8_t* const* valid) {
  FB_CHECK(nkeys >= 1 && nkeys <= FB_MAX_KEYS, "nkeys=%d out of range [1,%d]", nkeys, FB_MAX_KEYS);
  memset(&k, 0, sizeof(k));
  k.nkeys = nkeys;
  k.digit_shift = -1;
  for (int i = 0; i < nkeys; ++i) {
    FB_CHECK(widths[i] == 1 || widths[i] == 2 || widths[i] == 4 || widths[i] == 8,
             "key %d has unsupported width %d", i, widths[i]);
    FB_CHECK(ptrs[i] != nullptr, "key %d pointer is NULL", i);
    k.ptr[i] = ptrs[i];
    k.width[i] = widths[i];
    k.valid[i] = valid ? valid[i] : nullptr;
  }
  return 0;
}

struct PlanLayout {
  size_t hist_bytes;     // uint32 [nchunks][num]
  size_t pid_offset;     // rank records, kMetaBytes per full tile (num <= 256), 256-byte aligned
  size_t total_bytes;
};

PlanLayout plan_layout(const ChunkGeom& g, uint32_t num) {
  PlanLayout l;
  l.hist_bytes = (((size_t)g.nchunks * num * sizeof(uint32_t)) + 255) & ~(size_t)255;
  l.pid_offset = l.hist_bytes + 256;
  l.total_bytes = l.pid_offset + (num <= kSwcMaxNum ? (size_t)(g.full_rows / kTile) * kMetaBytes : 0) + 256;
  return l;
}

}  // namespace

extern "C" {

size_t fb_partition_scratch_bytes(int dev, int64_t nrows, uint32_t num_partitions) {
  if (nrows < 0 || num_partitions == 0) return 0;
  ChunkGeom g = make_geom(dev, nrows);
  return plan_layout(g, num_partitions).total_bytes;
}

int fb_partition_ids(int dev, void* stream, int64_t nrows, int nkeys, const void* const* key_ptrs,
                     const int32_t* key_widths, const uint8_t* const* key_valid,
                     uint32_t num_partitions, uint32_t* out_pids) {
  FB_CHECK(nrows >= 0, "nrows < 0");
  FB_CHECK(num_partitions >= 1, "num_partitions must be >= 1");
  if (nrows == 0) return 0;
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  FbKeys k;
  if (int rc = fill_keys(k, nkeys, key_ptrs, key_widths, key_valid)) return rc;
  FbDiv dv = fb_make_div(num_partitions);
  int64_t blocks = (nrows + 255) / 256;
  int64_t maxb = (int64_t)fb_sm_count(dev) * 16;
  if (blocks > maxb) blocks = maxb;
  cudaStream_t st = (cudaStream_t)stream;
  if (single_u64_key(nkeys, key_widths, key_valid))
    fb_pid_kernel<true><<<(unsigned)blocks, 256, 0, st>>>(k, dv, nrows, out_pids);
  else
    fb_pid_kernel<false><<<(unsigned)blocks, 256, 0, st>>>(k, dv, nrows, out_pids);
  FB_CUDA(cudaGetLastError());
  return 0;
}

int fb_row_hash64(int dev, void* stream, int64_t nrows, int nkeys, const void* const* key_ptrs,
                  const int32_t* key_widths, const uint8_t* const* key_valid, uint64_t* out_hash) {
  FB_CHECK(nrows >= 0, "nrows < 0");
  if (nrows == 0) return 0;
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  FbKeys k;
  if (int rc = fill_keys(k, nkeys, key_ptrs, key_widths, key_valid)) return rc;
  int64_t blocks = (nrows + 255) / 256;
  int64_t maxb = (int64_t)fb_sm_count(dev) * 16;
  if (blocks > maxb) blocks = maxb;
  fb_row_hash_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(k, nrows, out_hash);
  FB_CUDA(cudaGetLastError());
  return 0;
}

static int plan_impl(int dev, void* stream, int64_t nrows, const FbKeys& k, bool single,
                     uint32_t num_partitions, void* scratch, size_t scratch_bytes,
                     int64_t* out_part_offsets) {
  FB_CHECK(nrows >= 0, "nrows < 0");
  FB_CHECK(nrows < ((int64_t)1 << 32), "nrows=%lld exceeds the 2^32-1 rows one call handles",
           (long long)nrows);
  FB_CHECK(num_partitions >= 1 && num_partitions <= FB_MAX_PARTITIONS,
           "num_partitions=%u out of range [1,%d]", num_partitions, FB_MAX_PARTITIONS);
  FB_CHECK(out_part_offsets != nullptr, "out_part_offsets is NULL");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  cudaStream_t st = (cudaStream_t)stream;
  if (nrows == 0) {
    FB_CUDA(cudaMemsetAsync(out_part_offsets, 0, sizeof(int64_t) * ((size_t)num_partitions + 1), st));
    return 0;
  }
  ChunkGeom g = make_geom(dev, nrows);
  PlanLayout l = plan_layout(g, num_partitions);
  FB_CHECK(scratch != nullptr && scratch_bytes >= l.total_bytes,
           "scratch too small: need %zu bytes, got %zu", l.total_bytes, scratch_bytes);
  FbDiv dv = fb_make_div(num_partitions);
  uint32_t* hist = (uint32_t*)scratch;
  size_t smem = (size_t)kHistWarps * num_partitions * sizeof(uint32_t);
  FB_CUDA(ensure_smem_optin(dev));
  const int bits = bits_for(num_partitions);
  // num <= 256: full tiles are ranked completely (fb_rank_tile_kernel); the tail chunk and larger
  // partition counts only need the histogram
  int hist_chunk0 = 0;
  if (num_partitions <= kSwcMaxNum && g.nchunks_full > 0) {
    uint8_t* meta = (uint8_t*)scratch + l.pid_offset;
#define FB_LAUNCH_RANK(S, B, STAGED) \
  fb_rank_tile_kernel<S, B, STAGED><<<g.nchunks_full, kRankBlock, 0, st>>>(k, dv, num_partitions, g, hist, meta)
    if (single) {
      if (bits == 4) FB_LAUNCH_RANK(true, 4, true);
      else FB_LAUNCH_RANK(true, 8, true);
    } else if (k.digit_shift >= 0) {
      if (bits == 4) FB_LAUNCH_RANK(false, 4, true);
      else FB_LAUNCH_RANK(false, 8, true);
    } else {
      if (bits == 4) FB_LAUNCH_RANK(false, 4, false);
      else FB_LAUNCH_RANK(false, 8, false);
    }
#undef FB_LAUNCH_RANK
    FB_CUDA(cudaGetLastError());
    hist_chunk0 = g.nchunks_full;
  }
  if (hist_chunk0 < g.nchunks) {
#define FB_LAUNCH_HIST(S, B)                                                                       \
  fb_hist_kernel<S, B><<<g.nchunks - hist_chunk0, kHistBlock, smem, st>>>(k, dv, num_partitions, g, \
                                                                          hist_chunk0, hist)
    FB_DISPATCH_SB(single, bits, FB_LAUNCH_HIST);
#undef FB_LAUNCH_HIST
    FB_CUDA(cudaGetLastError());
  }
  fb_scan_chunks_kernel<<<num_partitions, 256, 0, st>>>(hist, num_partitions, g.nchunks, out_part_offsets);
  FB_CUDA(cudaGetLastError());
  fb_scan_parts_kernel<<<1, 1024, 0, st>>>(out_part_offsets, num_partitions);
  FB_CUDA(cudaGetLastError());
  return 0;
}

int fb_partition_plan(int dev, void* stream, int64_t nrows, int nkeys, const void* const* key_ptrs,
                      const int32_t* key_widths, const uint8_t* const* key_valid,
                      uint32_t num_partitions, void* scratch, size_t scratch_bytes,
                      int64_t* out_part_offsets) {
  FbKeys k;
  if (nrows == 0) {  // empty tables have NULL column pointers: nothing to read, offsets are all zero
    memset(&k, 0, sizeof(k));
    k.nkeys = 1;
    k.digit_shift = -1;
    return plan_impl(dev, stream, 0, k, false, num_partitions, scratch, scratch_bytes, out_part_offsets);
  }
  if (int rc = fill_keys(k, nkeys, key_ptrs, key_widths, key_valid)) return rc;
  return plan_impl(dev, stream, nrows, k, single_u64_key(nkeys, key_widths, key_valid), num_partitions,
                   scratch, scratch_bytes, out_part_offsets);
}

// Rows of the partial tail tile of the mapped units, evaluated into tail_tmp[c][0 .. nrows - full_rows): the
// generic scatter kernel then moves them like any column.
__global__ void fb_map_tail_kernel(int ncols, const void* const* __restrict__ x_ptrs, const fb_map_unit* __restrict__ maps,
                                   int64_t row0, int64_t nrows, uint64_t* __restrict__ tmp) {
  const int64_t n = nrows - row0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * ncols; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / n);
    const int64_t r = row0 + i % n;
    const fb_map_unit m = maps[c];
    const uint64_t x = ((const uint64_t*)x_ptrs[c])[r];
    const uint64_t y = m.src2 != nullptr ? ((const uint64_t*)m.src2)[r] : 0;
    tmp[(size_t)c * kTile + (size_t)(i % n)] = ws_apply_map(m.mode, m.src2 != nullptr, x, y, m.a, m.b, m.c);
  }
}

static int apply_impl(int dev, void* stream, int64_t nrows, const FbKeys& k, bool single,
                      uint32_t num_partitions, const void* scratch, size_t scratch_bytes,
                      const int64_t* part_offsets, int ncols, const void* const* col_ptrs,
                      const int32_t* col_widths, void* const* out_col_ptrs, int sm_reserve = 0,
                      const fb_map_unit* maps = nullptr, void* tail_tmp = nullptr, int cols_per_launch_req = 0) {
  FB_CHECK(nrows >= 0 && nrows < ((int64_t)1 << 32), "nrows out of range");
  FB_CHECK(num_partitions >= 1 && num_partitions <= FB_MAX_PARTITIONS,
           "num_partitions=%u out of range [1,%d]", num_partitions, FB_MAX_PARTITIONS);
  FB_CHECK(ncols >= 0, "ncols < 0");
  if (nrows == 0 || ncols == 0) return 0;
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  ChunkGeom g = make_geom(dev, nrows);
  PlanLayout l = plan_layout(g, num_partitions);
  FB_CHECK(scratch != nullptr && scratch_bytes >= l.total_bytes, "scratch too small");
  FbDiv dv = fb_make_div(num_partitions);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = scatter_smem_bytes(num_partitions);
  FB_CUDA(ensure_smem_optin(dev));
  const int bits = bits_for(num_partitions);

  for (int c = 0; c < ncols; ++c) {
    const int w = col_widths[c];
    FB_CHECK(w == 1 || w == 2 || w == 4 || w == 8, "column %d has unsupported width %d", c, w);
    FB_CHECK(col_ptrs[c] != nullptr && out_col_ptrs[c] != nullptr, "column %d pointer is NULL", c);
  }

  // generic kernel over chunks [chunk0, chunk0 + nch) for the columns listed in idx[0..n)
  const void* const* gen_src = col_ptrs;
  auto launch_generic = [&](const int* idx, int n, int chunk0, int nch) -> int {
    for (int c0 = 0; c0 < n && nch > 0; c0 += FB_MAX_COLS) {
      FbCols cols;
      memset(&cols, 0, sizeof(cols));
      cols.ncols = n - c0 < FB_MAX_COLS ? n - c0 : FB_MAX_COLS;
      bool all8 = true;
      for (int c = 0; c < cols.ncols; ++c) {
        cols.src[c] = gen_src[idx[c0 + c]];
        cols.dst[c] = out_col_ptrs[idx[c0 + c]];
        cols.width[c] = col_widths[idx[c0 + c]];
        all8 = all8 && cols.width[c] == 8;
      }
#define FB_LAUNCH_SCATTER(S, B)                                                                        \
  do {                                                                                                 \
    if (all8)                                                                                          \
      fb_scatter_kernel<S, B, true><<<nch, kBlock, smem, st>>>(k, dv, num_partitions, g, chunk0,       \
                                                               (const uint32_t*)scratch, part_offsets, cols); \
    else                                                                                               \
      fb_scatter_kernel<S, B, false><<<nch, kBlock, smem, st>>>(k, dv, num_partitions, g, chunk0,      \
                                                                (const uint32_t*)scratch, part_offsets, cols); \
  } while (0)
      FB_DISPATCH_SB(single, bits, FB_LAUNCH_SCATTER);
#undef FB_LAUNCH_SCATTER
      FB_CUDA(cudaGetLastError());
    }
    return 0;
  };

  // ---- split the columns: fast path (warp-specialised TMA ring + write combining; reads the rank
  //      records written by pass 1, so any key shape qualifies) vs generic.  8-byte columns, num <= 256.
  const bool fast_ok = num_partitions <= kSwcMaxNum && g.nchunks_full > 0;
  if (maps != nullptr) {  // fused map epilogue (K4): every unit must qualify for the fast kernel
    FB_CHECK(num_partitions <= kSwcMaxNum, "fused map needs num_partitions <= %u", kSwcMaxNum);
    FB_CHECK(tail_tmp != nullptr || g.full_rows == nrows, "fused map: tail_tmp is NULL");
    for (int c = 0; c < ncols; ++c) {
      FB_CHECK(col_widths[c] == 8 && (uintptr_t)col_ptrs[c] % 16 == 0, "fused map: column %d is not an aligned 8-byte column", c);
      FB_CHECK(maps[c].mode >= 0 && maps[c].mode <= 2, "fused map: column %d has mode %d", c, maps[c].mode);
      FB_CHECK(maps[c].src2 == nullptr || (maps[c].mode != 0 && (uintptr_t)maps[c].src2 % 16 == 0),
               "fused map: bad second operand of column %d", c);
    }
  }
  int* fast_idx = (int*)alloca(sizeof(int) * (size_t)ncols);
  int* gen_idx = (int*)alloca(sizeof(int) * (size_t)ncols);
  int nfast = 0, ngen = 0;
  for (int c = 0; c < ncols; ++c) {
    if (fast_ok && col_widths[c] == 8 && (uintptr_t)col_ptrs[c] % 16 == 0) fast_idx[nfast++] = c;
    else gen_idx[ngen++] = c;
  }
  if (int rc = launch_generic(gen_idx, ngen, 0, g.nchunks)) return rc;

  if (nfast > 0) {
    int smem_max = 0;
    FB_CUDA(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    // sm_reserve: SMs left free for kernels that must co-run with this persistent one (the
    // multi-GPU barrier / pull kernels: a scatter CTA owns the whole register file of its SM)
    int avail = fb_sm_count(dev) - sm_reserve;
    if (avail < 1) avail = 1;
    const uint8_t* pid_plane = (const uint8_t*)scratch + l.pid_offset;  // rank records of pass 1
    // Column groups of at most 2, evenly sized.  Measured on H100 (100 M rows x 8 cols; MEASUREMENTS.md), one
    // launch per group at 700 W: 8 columns per group -> 6.54 ms, 4 -> 6.28, 3 -> 6.00, 2 -> 5.84, 1 -> 6.29; one
    // launch at 400 W: 4 -> 6.25, 2 -> 5.56, 1 -> 5.88 (all with 4-row write groups: with more than 2 columns in
    // flight per CTA, half-written lines no longer met their other half in the 50 MB L2).  With whole-line groups
    // at 2 columns, one launch at 700 W: 2 -> 5.04 ms, against 5.39 for 1 column per group at G = 4.
    int ngroups = (nfast + 1) / 2;
    int per_group = (nfast + ngroups - 1) / ngroups;
    if (cols_per_launch_req >= 1 && cols_per_launch_req <= kSwcMaxCols) per_group = cols_per_launch_req;
    ngroups = (nfast + per_group - 1) / per_group;
    const size_t stage_bytes = (size_t)kWsRankers * kWsRankItems * 8;
    auto stages_for = [&](size_t book) { return book < (size_t)smem_max ? (int)(((size_t)smem_max - book) / stage_bytes) : 0; };
    // Whole-line groups (kWsG) for groups of 2 columns, if the ring keeps kWsMinStages stages next to their carry.
    // H100 at 700 W, one launch, 100 M rows x 8 columns (MEASUREMENTS.md): 2 columns per group 5.31 ms at G = 4,
    // 5.18 at G = 8, 5.04 at G = 16; 1 column per group 5.39 at G = 4, 6.03 at G = 16 (the rankers' longer
    // per-tile work at G = 16 is no longer hidden behind the moves of a single column).
    const bool lines = per_group == 2 &&
                       stages_for(ws_book_bytes<kWsG, kWsRankItems>(num_partitions, per_group)) >= kWsMinStages;
    const size_t book = lines ? ws_book_bytes<kWsG, kWsRankItems>(num_partitions, per_group)
                              : ws_book_bytes<kWsGWide, kWsRankItems>(num_partitions, per_group);
    int nstages = stages_for(book);
    if (nstages > 16) nstages = 16;
    FB_CHECK(nstages >= 2, "not enough shared memory for the TMA ring (%d stages)", nstages);
    const size_t tsmem = (size_t)nstages * stage_bytes + book;
    // All groups in one launch of ngroups x S CTAs, the ngroups CTAs of a chunk side by side (WsUnits), up to
    // FB_MAX_COLS units per launch.  With fewer free SMs than groups: one launch per group, over all chunks.
    const int groups_per_launch = ngroups <= avail ? (ngroups < FB_MAX_COLS / per_group ? ngroups : FB_MAX_COLS / per_group) : 1;
    for (int g0 = 0; g0 < ngroups; g0 += groups_per_launch) {
      const int lg = ngroups - g0 < groups_per_launch ? ngroups - g0 : groups_per_launch;
      const int c0 = g0 * per_group;
      const int nu = nfast - c0 < lg * per_group ? nfast - c0 : lg * per_group;
      WsUnits wu;
      WsMap wm;
      memset(&wu, 0, sizeof(wu));
      memset(&wm, 0, sizeof(wm));
      wu.nunits = nu;
      wu.per_group = per_group;
      wu.ngroups = lg;
      for (int c = 0; c < nu; ++c) {
        wu.src[c] = (const uint64_t*)col_ptrs[fast_idx[c0 + c]];
        wu.dst[c] = (uint64_t*)out_col_ptrs[fast_idx[c0 + c]];
        if (maps != nullptr) {
          const fb_map_unit& m = maps[fast_idx[c0 + c]];
          wm.src2[c] = (const uint64_t*)m.src2;
          wm.a[c] = m.a; wm.b[c] = m.b; wm.c[c] = m.c;
          wm.mode[c] = m.mode;
        }
      }
      const int64_t ctas = avail < (int64_t)lg * g.nchunks_full ? avail : (int64_t)lg * g.nchunks_full;
      const int grid = (int)(ctas / lg) * lg;
#define FB_LAUNCH_WS(B, G, M)                                                                               \
  fb_scatter_ws_kernel<B, G, kWsRankItems, M><<<grid, kWsThreads, tsmem, st>>>(                              \
      wu, num_partitions, g, nstages, pid_plane, (const uint32_t*)scratch, part_offsets, wm)
#define FB_LAUNCH_WS_G(G)                                                                                   \
  do {                                                                                                      \
    if (maps != nullptr) {                                                                                  \
      if (bits == 4) FB_LAUNCH_WS(4, G, true);                                                              \
      else FB_LAUNCH_WS(8, G, true);                                                                        \
    } else if (bits == 4) {                                                                                 \
      FB_LAUNCH_WS(4, G, false);                                                                            \
    } else {                                                                                                \
      FB_LAUNCH_WS(8, G, false);                                                                            \
    }                                                                                                       \
  } while (0)
      if (lines) FB_LAUNCH_WS_G(kWsG);
      else FB_LAUNCH_WS_G(kWsGWide);
#undef FB_LAUNCH_WS_G
#undef FB_LAUNCH_WS
      FB_CUDA(cudaGetLastError());
    }
    // the partial tail tile of the fast columns
    if (maps == nullptr)
      if (int rc = launch_generic(fast_idx, nfast, g.nchunks_full, g.nchunks - g.nchunks_full)) return rc;
  }
  if (maps != nullptr && g.full_rows < nrows) {
    // fused map: the tail rows are mapped into tail_tmp (device arrays of pointers / descriptors live in
    // its first bytes) and the generic kernel reads them through shifted column bases
    FB_CHECK(ncols <= kSwcMaxCols * 8, "fused map: too many columns (%d)", ncols);
    uint8_t* base = (uint8_t*)tail_tmp;
    const size_t hdr = (((size_t)ncols * (sizeof(void*) + sizeof(fb_map_unit))) + 255) & ~(size_t)255;
    FB_CUDA(cudaMemcpyAsync(base, col_ptrs, sizeof(void*) * (size_t)ncols, cudaMemcpyHostToDevice, st));
    FB_CUDA(cudaMemcpyAsync(base + sizeof(void*) * (size_t)ncols, maps, sizeof(fb_map_unit) * (size_t)ncols,
                            cudaMemcpyHostToDevice, st));
    uint64_t* vals = (uint64_t*)(base + hdr);
    fb_map_tail_kernel<<<32, 256, 0, st>>>(ncols, (const void* const*)base,
                                           (const fb_map_unit*)(base + sizeof(void*) * (size_t)ncols), g.full_rows,
                                           nrows, vals);
    FB_CUDA(cudaGetLastError());
    const void** shifted = (const void**)alloca(sizeof(void*) * (size_t)ncols);
    int* all_idx = (int*)alloca(sizeof(int) * (size_t)ncols);
    for (int c = 0; c < ncols; ++c) {
      shifted[c] = (const uint8_t*)(vals + (size_t)c * kTile) - (size_t)g.full_rows * 8;
      all_idx[c] = c;
    }
    gen_src = shifted;
    if (int rc = launch_generic(all_idx, ncols, g.nchunks_full, g.nchunks - g.nchunks_full)) return rc;
  }
  return 0;
}

int fb_partition_apply(int dev, void* stream, int64_t nrows, int nkeys, const void* const* key_ptrs,
                       const int32_t* key_widths, const uint8_t* const* key_valid,
                       uint32_t num_partitions, const void* scratch, size_t scratch_bytes,
                       const int64_t* part_offsets, int ncols, const void* const* col_ptrs,
                       const int32_t* col_widths, void* const* out_col_ptrs) {
  if (nrows == 0 || ncols == 0) return 0;
  FbKeys k;
  if (int rc = fill_keys(k, nkeys, key_ptrs, key_widths, key_valid)) return rc;
  return apply_impl(dev, stream, nrows, k, single_u64_key(nkeys, key_widths, key_valid), num_partitions,
                    scratch, scratch_bytes, part_offsets, ncols, col_ptrs, col_widths, out_col_ptrs);
}

int fb_partition_apply_ex(int dev, void* stream, int64_t nrows, int nkeys, const void* const* key_ptrs,
                          const int32_t* key_widths, const uint8_t* const* key_valid,
                          uint32_t num_partitions, const void* scratch, size_t scratch_bytes,
                          const int64_t* part_offsets, int ncols, const void* const* col_ptrs,
                          const int32_t* col_widths, void* const* out_col_ptrs, int sm_reserve,
                          int cols_per_launch) {
  if (nrows == 0 || ncols == 0) return 0;
  FB_CHECK(sm_reserve >= 0, "sm_reserve < 0");
  FbKeys k;
  if (int rc = fill_keys(k, nkeys, key_ptrs, key_widths, key_valid)) return rc;
  return apply_impl(dev, stream, nrows, k, single_u64_key(nkeys, key_widths, key_valid), num_partitions,
                    scratch, scratch_bytes, part_offsets, ncols, col_ptrs, col_widths, out_col_ptrs, sm_reserve,
                    nullptr, nullptr, cols_per_launch);
}

size_t fb_partition_map_tail_bytes(int ncols) {
  if (ncols < 0) return 0;
  return ((((size_t)ncols * (sizeof(void*) + sizeof(fb_map_unit))) + 255) & ~(size_t)255) + (size_t)ncols * kTile * 8;
}

int fb_partition_apply_map(int dev, void* stream, int64_t nrows, int nkeys, const void* const* key_ptrs,
                           const int32_t* key_widths, const uint8_t* const* key_valid,
                           uint32_t num_partitions, const void* scratch, size_t scratch_bytes,
                           const int64_t* part_offsets, int ncols, const void* const* col_ptrs,
                           void* const* out_col_ptrs, const fb_map_unit* maps, void* tail_tmp, int sm_reserve) {
  if (nrows == 0 || ncols == 0) return 0;
  FB_CHECK(maps != nullptr, "maps is NULL");
  FB_CHECK(ncols <= FB_MAX_COLS, "ncols=%d > %d", ncols, FB_MAX_COLS);
  FbKeys k;
  if (int rc = fill_keys(k, nkeys, key_ptrs, key_widths, key_valid)) return rc;
  int32_t widths[FB_MAX_COLS];
  for (int c = 0; c < ncols; ++c) widths[c] = 8;
  return apply_impl(dev, stream, nrows, k, single_u64_key(nkeys, key_widths, key_valid), num_partitions,
                    scratch, scratch_bytes, part_offsets, ncols, col_ptrs, widths, out_col_ptrs, sm_reserve, maps,
                    tail_tmp);
}

int fb_radix_pass(int dev, void* stream, int64_t nrows, const void* sort_key_u64, int shift, int ncols,
                  const void* const* col_ptrs, const int32_t* col_widths, void* const* out_col_ptrs,
                  void* scratch, size_t scratch_bytes, int64_t* d_offsets /*257*/) {
  FB_CHECK(shift >= 0 && shift <= 56, "shift out of range");
  if (nrows == 0) return 0;
  const void* kp[1] = {sort_key_u64};
  const int32_t kw[1] = {8};
  FbKeys k;
  if (int rc = fill_keys(k, 1, kp, kw, nullptr)) return rc;
  k.digit_shift = shift;
  if (int rc = plan_impl(dev, stream, nrows, k, false, 256, scratch, scratch_bytes, d_offsets)) return rc;
  return apply_impl(dev, stream, nrows, k, false, 256, scratch, scratch_bytes, d_offsets, ncols, col_ptrs,
                    col_widths, out_col_ptrs);
}

int fb_partition_cols(int dev, void* stream, int64_t nrows, int ncols, const void* const* col_ptrs,
                      const int32_t* col_widths, const int32_t* key_col_idx, int nkeys,
                      const uint8_t* const* key_valid, uint32_t num_partitions,
                      void* const* out_col_ptrs, int64_t* out_part_offsets, void* scratch,
                      size_t scratch_bytes) {
  FB_CHECK(nkeys >= 1 && nkeys <= FB_MAX_KEYS, "nkeys=%d out of range [1,%d]", nkeys, FB_MAX_KEYS);
  const void* kp[FB_MAX_KEYS];
  int32_t kw[FB_MAX_KEYS];
  for (int i = 0; i < nkeys; ++i) {
    FB_CHECK(key_col_idx[i] >= 0 && key_col_idx[i] < ncols, "key column index %d out of range", key_col_idx[i]);
    kp[i] = col_ptrs[key_col_idx[i]];
    kw[i] = col_widths[key_col_idx[i]];
  }
  if (int rc = fb_partition_plan(dev, stream, nrows, nkeys, kp, kw, key_valid, num_partitions, scratch,
                                 scratch_bytes, out_part_offsets))
    return rc;
  return fb_partition_apply(dev, stream, nrows, nkeys, kp, kw, key_valid, num_partitions, scratch,
                            scratch_bytes, out_part_offsets, ncols, col_ptrs, col_widths, out_col_ptrs);
}

int fb_bits_to_bytes(int dev, void* stream, const uint8_t* bits, int64_t bit_offset, int64_t nrows,
                     uint8_t* out_bytes) {
  if (nrows <= 0) return 0;
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  int64_t blocks = (nrows + 255) / 256;
  if (blocks > fb_sm_count(dev) * 16) blocks = fb_sm_count(dev) * 16;
  fb_bits_to_bytes_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(bits, bit_offset, nrows, out_bytes);
  FB_CUDA(cudaGetLastError());
  return 0;
}

int fb_bytes_to_bits(int dev, void* stream, const uint8_t* bytes, int64_t nrows, uint8_t* out_bits,
                     int64_t* out_null_count) {
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  cudaStream_t st = (cudaStream_t)stream;
  if (out_null_count) FB_CUDA(cudaMemsetAsync(out_null_count, 0, sizeof(int64_t), st));
  if (nrows <= 0) return 0;
  int64_t nbytes = (nrows + 7) / 8;
  int64_t blocks = (nbytes + 255) / 256;
  if (blocks > fb_sm_count(dev) * 16) blocks = fb_sm_count(dev) * 16;
  fb_bytes_to_bits_kernel<<<(unsigned)blocks, 256, 0, st>>>(bytes, nrows, out_bits,
                                                           (unsigned long long*)out_null_count);
  FB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
