// K12 string-building functions for sm_90a, evaluated once per dictionary entry (include/fugue_b200.h).
//
// UPPER, LOWER, SUBSTR, TRIM, REPLACE and concatenation of one string column depend on the dictionary entry
// alone, so they run over the entries and build a new dictionary.  fb_string_transform is called twice per
// function: the measure call writes every output's byte length and validity, the host scans the lengths into
// offsets, and the write call fills the bytes.  Both calls run the same per-entry code (an emitter that only
// counts, or one that also stores), so the lengths and the bytes cannot disagree.
//
// Equal results must share one code (K6 grouping, ranks and set operations assume distinct entries), so the
// host deduplicates: fb_string_hash, the radix sort of (hash, entry) pairs, then fb_string_first_equal gives
// every entry the smallest entry id with equal bytes.  The kept entries are gathered by a write call with a
// source list.
//
// One thread per entry, grid-stride.  Literal arguments and FORMAT tokens are a kernel parameter (constant
// bank).  UPPER / LOWER map ASCII in registers and other code points by a binary search in the sorted
// (from, to) table of fb_casemap.inc, staged in shared memory.
#include "fb_common.cuh"
#include "fb_casemap.inc"

namespace {

constexpr int kThreads = 256;
constexpr int64_t kNoLength = (int64_t)1 << 62;  // SUBSTR without a length: every code point after start

struct StrProgram {
  int32_t op, null_is_empty, has_length, ntok;
  int64_t start, length;
  int32_t nlit[2];
  uint8_t lit[2][FB_STR_MAX_LITERAL];
  int16_t tok[FB_STR_MAX_TOKENS];
};
static_assert(sizeof(StrProgram) <= 4000, "the program must fit the kernel parameter space");

__device__ __forceinline__ bool is_cont(uint8_t b) { return (b & 0xC0) == 0x80; }

// the end of the code point that starts at byte i of s[0, len): the next byte that is not a continuation byte
__device__ __forceinline__ int64_t cp_end(const uint8_t* __restrict__ s, int64_t len, int64_t i) {
  ++i;
  while (i < len && is_cont(s[i])) ++i;
  return i;
}

// counts the output bytes; the writing emitter also stores them
template <bool kWrite>
struct Emit {
  uint8_t* __restrict__ out;
  int64_t n = 0;
  __device__ __forceinline__ void put(uint8_t b) {
    if (kWrite) out[n] = b;
    ++n;
  }
  __device__ __forceinline__ void put(const uint8_t* __restrict__ p, int64_t k) {
    if (kWrite)
      for (int64_t j = 0; j < k; ++j) out[n + j] = p[j];
    n += k;
  }
};

template <typename E>
__device__ __forceinline__ void put_cp(E& e, uint32_t c) {
  if (c < 0x80) {
    e.put((uint8_t)c);
  } else if (c < 0x800) {
    e.put((uint8_t)(0xC0 | (c >> 6)));
    e.put((uint8_t)(0x80 | (c & 0x3F)));
  } else if (c < 0x10000) {
    e.put((uint8_t)(0xE0 | (c >> 12)));
    e.put((uint8_t)(0x80 | ((c >> 6) & 0x3F)));
    e.put((uint8_t)(0x80 | (c & 0x3F)));
  } else {
    e.put((uint8_t)(0xF0 | (c >> 18)));
    e.put((uint8_t)(0x80 | ((c >> 12) & 0x3F)));
    e.put((uint8_t)(0x80 | ((c >> 6) & 0x3F)));
    e.put((uint8_t)(0x80 | (c & 0x3F)));
  }
}

// UPPER / LOWER: every well-formed code point through the table; any other byte is copied as it is
template <typename E>
__device__ void case_map(E& e, const uint8_t* __restrict__ s, int64_t len, bool upper, const uint2* __restrict__ map,
                         int nmap) {
  for (int64_t i = 0; i < len;) {
    const uint8_t b = s[i];
    if (b < 0x80) {
      e.put(upper ? (b >= 'a' && b <= 'z' ? b - 32 : b) : (b >= 'A' && b <= 'Z' ? b + 32 : b));
      ++i;
      continue;
    }
    const int k = b >= 0xF0 ? 4 : (b >= 0xE0 ? 3 : (b >= 0xC0 ? 2 : 0));
    bool ok = k > 0 && i + k <= len;
    uint32_t c = k == 4 ? (b & 0x07) : (k == 3 ? (b & 0x0F) : (b & 0x1F));
    for (int j = 1; ok && j < k; ++j) {
      ok = is_cont(s[i + j]);
      c = (c << 6) | (s[i + j] & 0x3F);
    }
    if (!ok) {  // not UTF-8: keep the byte
      e.put(b);
      ++i;
      continue;
    }
    int lo = 0, hi = nmap;  // the first entry whose source is >= c
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (map[mid].x < c) lo = mid + 1; else hi = mid;
    }
    if (lo < nmap && map[lo].x == c) put_cp(e, map[lo].y);
    else e.put(s + i, k);
    i += k;
  }
}

// SQLite's substr(s, start, length) in code points (func.c substrFunc)
template <typename E>
__device__ void substr(E& e, const StrProgram& P, const uint8_t* __restrict__ s, int64_t len) {
  int64_t p1 = P.start, p2 = P.has_length ? P.length : kNoLength;
  bool neg = false;
  if (p2 < 0) {
    p2 = -p2;
    neg = true;
  }
  if (p1 < 0) {
    int64_t cps = 0;
    for (int64_t i = 0; i < len; ++i) cps += !is_cont(s[i]);
    p1 += cps;
    if (p1 < 0) {
      p2 += p1;
      if (p2 < 0) p2 = 0;
      p1 = 0;
    }
  } else if (p1 > 0) {
    --p1;
  } else if (p2 > 0) {
    --p2;
  }
  if (neg) {
    p1 -= p2;
    if (p1 < 0) {
      p2 += p1;
      p1 = 0;
    }
  }
  int64_t a = 0;
  for (; p1 > 0 && a < len; --p1) a = cp_end(s, len, a);
  int64_t b = a;
  for (; p2 > 0 && b < len; --p2) b = cp_end(s, len, b);
  e.put(s + a, b - a);
}

// is the code point s[a, b) one of the code points of literal 0?
__device__ __forceinline__ bool in_set(const StrProgram& P, const uint8_t* __restrict__ s, int64_t a, int64_t b) {
  const int n = P.nlit[0];
  for (int i = 0; i < n;) {
    const int j = (int)cp_end(P.lit[0], n, i);
    bool eq = j - i == b - a;
    for (int k = 0; eq && k < j - i; ++k) eq = P.lit[0][i + k] == s[a + k];
    if (eq) return true;
    i = j;
  }
  return false;
}

template <typename E>
__device__ void trim(E& e, const StrProgram& P, const uint8_t* __restrict__ s, int64_t len) {
  int64_t a = 0, b = len;
  if (P.op != FB_STR_RTRIM) {
    while (a < b) {
      const int64_t c = cp_end(s, b, a);
      if (!in_set(P, s, a, c)) break;
      a = c;
    }
  }
  if (P.op != FB_STR_LTRIM) {
    while (b > a) {
      int64_t c = b - 1;
      while (c > a && is_cont(s[c])) --c;
      if (!in_set(P, s, c, b)) break;
      b = c;
    }
  }
  e.put(s + a, b - a);
}

// SQLite's replace: non-overlapping matches of literal 0, left to right, each replaced by literal 1
template <typename E>
__device__ void replace(E& e, const StrProgram& P, const uint8_t* __restrict__ s, int64_t len) {
  const int nf = P.nlit[0];
  if (nf == 0) {
    e.put(s, len);
    return;
  }
  const uint8_t f0 = P.lit[0][0];
  int64_t i = 0;
  while (i < len) {
    bool hit = s[i] == f0 && i + nf <= len;
    for (int k = 1; hit && k < nf; ++k) hit = s[i + k] == P.lit[0][k];
    if (hit) {
      e.put(P.lit[1], P.nlit[1]);
      i += nf;
    } else {
      e.put(s[i]);
      ++i;
    }
  }
}

// the result of entry (s, len, ok) into e; returns its validity
template <typename E>
__device__ bool entry(E& e, const StrProgram& P, const uint8_t* __restrict__ s, int64_t len, bool ok,
                      const uint2* __restrict__ map, int nmap) {
  if (P.op == FB_STR_FORMAT) {
    if (!ok && !P.null_is_empty) return false;
    for (int t = 0; t < P.ntok; ++t) {
      const int tk = P.tok[t];
      if (tk == FB_STR_SELF) {
        if (ok) e.put(s, len);
      } else {
        e.put((uint8_t)tk);
      }
    }
    return true;
  }
  if (!ok) return false;
  switch (P.op) {
    case FB_STR_COPY: e.put(s, len); break;
    case FB_STR_UPPER: case_map(e, s, len, true, map, nmap); break;
    case FB_STR_LOWER: case_map(e, s, len, false, map, nmap); break;
    case FB_STR_SUBSTR: substr(e, P, s, len); break;
    case FB_STR_REPLACE: replace(e, P, s, len); break;
    default: trim(e, P, s, len); break;
  }
  return true;
}

__global__ void __launch_bounds__(kThreads)
fb_string_transform_kernel(const __grid_constant__ StrProgram P, int64_t n, const int64_t* __restrict__ offsets,
                           const uint8_t* __restrict__ data, const uint8_t* __restrict__ valid,
                           const int64_t* __restrict__ src, int64_t* __restrict__ out_len,
                           uint8_t* __restrict__ out_valid, const int64_t* __restrict__ out_offsets,
                           uint8_t* __restrict__ out_data) {
  extern __shared__ uint2 s_map[];
  int nmap = 0;
  if (P.op == FB_STR_UPPER || P.op == FB_STR_LOWER) {
    const bool up = P.op == FB_STR_UPPER;
    nmap = up ? FB_CASEMAP_UPPER_N : FB_CASEMAP_LOWER_N;
    const unsigned int(*tab)[2] = up ? fb_casemap_upper : fb_casemap_lower;
    for (int j = threadIdx.x; j < nmap; j += kThreads) s_map[j] = make_uint2(tab[j][0], tab[j][1]);
    __syncthreads();
  }
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const int64_t k = src == nullptr ? i : src[i];
    const bool ok = valid == nullptr || valid[k] != 0;
    const int64_t a = offsets[k];
    if (out_data == nullptr) {
      Emit<false> e{nullptr};
      const bool v = entry(e, P, data + a, offsets[k + 1] - a, ok, s_map, nmap);
      out_len[i] = v ? e.n : 0;
      out_valid[i] = v ? 1 : 0;
    } else {
      Emit<true> e{out_data + out_offsets[i]};
      entry(e, P, data + a, offsets[k + 1] - a, ok, s_map, nmap);
    }
  }
}

// FNV-1a over the bytes, finished by the murmur3 64-bit mixer so that the low bits are well spread
__global__ void __launch_bounds__(kThreads)
fb_string_hash_kernel(int64_t n, const int64_t* __restrict__ offsets, const uint8_t* __restrict__ data,
                      const uint8_t* __restrict__ valid, uint64_t mask, uint64_t* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    uint64_t h = 0;
    if (valid == nullptr || valid[i] != 0) {
      const int64_t a = offsets[i], b = offsets[i + 1];
      h = 0xCBF29CE484222325ULL ^ (uint64_t)(b - a);
      for (int64_t p = a; p < b; ++p) h = (h ^ data[p]) * 0x100000001B3ULL;
      h ^= h >> 33;
      h *= 0xFF51AFD7ED558CCDULL;
      h ^= h >> 33;
      h *= 0xC4CEB9FE1A85EC53ULL;
      h ^= h >> 33;
    }
    out[i] = h & mask;
  }
}

__device__ __forceinline__ bool same_entry(const int64_t* __restrict__ offsets, const uint8_t* __restrict__ data,
                                           const uint8_t* __restrict__ valid, int64_t x, int64_t y) {
  const bool vx = valid == nullptr || valid[x] != 0, vy = valid == nullptr || valid[y] != 0;
  if (!vx || !vy) return vx == vy;
  const int64_t ax = offsets[x], ay = offsets[y], len = offsets[x + 1] - ax;
  if (offsets[y + 1] - ay != len) return false;
  for (int64_t j = 0; j < len; ++j)
    if (data[ax + j] != data[ay + j]) return false;
  return true;
}

__global__ void __launch_bounds__(kThreads)
fb_string_first_equal_kernel(int64_t n, const int64_t* __restrict__ offsets, const uint8_t* __restrict__ data,
                             const uint8_t* __restrict__ valid, const uint64_t* __restrict__ hash,
                             const int64_t* __restrict__ idx, int64_t* __restrict__ canon) {
  for (int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x; p < n; p += (int64_t)gridDim.x * kThreads) {
    const uint64_t h = hash[p];
    int64_t lo = 0, hi = p;  // the start of p's hash run: the first position whose hash is h
    while (lo < hi) {
      const int64_t mid = lo + ((hi - lo) >> 1);
      if (hash[mid] < h) lo = mid + 1; else hi = mid;
    }
    const int64_t e = idx[p];
    int64_t q = lo;
    while (q < p && !same_entry(offsets, data, valid, idx[q], e)) ++q;
    canon[e] = idx[q];
  }
}

unsigned grid_for(int dev, int64_t n) {
  const int64_t blocks = (n + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)fb_sm_count(dev) * 8;
  return (unsigned)(blocks < cap ? blocks : cap);
}

}  // namespace

extern "C" int fb_string_transform(int dev, void* stream, int op, int64_t n, const int64_t* offsets,
                                   const uint8_t* data, const uint8_t* valid, const int64_t* src, int64_t start,
                                   int64_t length, int has_length, int nlit0, const uint8_t* lit0, int nlit1,
                                   const uint8_t* lit1, int ntokens, const int16_t* tokens, int null_is_empty,
                                   int64_t* out_len, uint8_t* out_valid, const int64_t* out_offsets,
                                   uint8_t* out_data) {
  FB_CHECK(n >= 0, "n < 0");
  FB_CHECK(op >= FB_STR_COPY && op <= FB_STR_FORMAT, "unknown op %d", op);
  FB_CHECK(nlit0 >= 0 && nlit0 <= FB_STR_MAX_LITERAL && nlit1 >= 0 && nlit1 <= FB_STR_MAX_LITERAL,
           "literal of %d / %d bytes; at most %d", nlit0, nlit1, FB_STR_MAX_LITERAL);
  FB_CHECK((nlit0 == 0 || lit0 != nullptr) && (nlit1 == 0 || lit1 != nullptr), "NULL literal");
  FB_CHECK(ntokens >= 0 && ntokens <= FB_STR_MAX_TOKENS, "ntokens=%d out of range [0,%d]", ntokens,
           FB_STR_MAX_TOKENS);
  FB_CHECK(ntokens == 0 || tokens != nullptr, "NULL tokens");
  FB_CHECK(op != FB_STR_SUBSTR || (start >= -kNoLength && start <= kNoLength &&
                                   (!has_length || (length >= -kNoLength && length <= kNoLength))),
           "SUBSTR start / length outside [-2^62, 2^62]");
  StrProgram P;
  memset(&P, 0, sizeof(P));
  P.op = op;
  P.null_is_empty = null_is_empty != 0;
  P.has_length = has_length != 0;
  P.start = start;
  P.length = length;
  P.nlit[0] = nlit0;
  P.nlit[1] = nlit1;
  if (nlit0) memcpy(P.lit[0], lit0, nlit0);
  if (nlit1) memcpy(P.lit[1], lit1, nlit1);
  for (int t = 0; t < ntokens; ++t) {
    FB_CHECK(tokens[t] >= 0 && tokens[t] <= FB_STR_SELF, "token %d: unknown value %d", t, (int)tokens[t]);
    P.tok[t] = tokens[t];
  }
  P.ntok = ntokens;
  if (n == 0) return 0;
  FB_CHECK(offsets != nullptr && data != nullptr, "NULL dictionary");
  FB_CHECK(out_data != nullptr ? out_offsets != nullptr : (out_len != nullptr && out_valid != nullptr),
           "NULL output");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  size_t smem = 0;
  if (op == FB_STR_UPPER) smem = sizeof(uint2) * FB_CASEMAP_UPPER_N;
  if (op == FB_STR_LOWER) smem = sizeof(uint2) * FB_CASEMAP_LOWER_N;
  fb_string_transform_kernel<<<grid_for(dev, n), kThreads, smem, (cudaStream_t)stream>>>(
      P, n, offsets, data, valid, src, out_len, out_valid, out_offsets, out_data);
  FB_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int fb_string_hash(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                              const uint8_t* valid, int bits, uint64_t* out) {
  FB_CHECK(n >= 0, "n < 0");
  FB_CHECK(bits >= 1 && bits <= 64, "bits=%d out of range [1,64]", bits);
  if (n == 0) return 0;
  FB_CHECK(offsets != nullptr && data != nullptr && out != nullptr, "NULL argument");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  const uint64_t mask = bits == 64 ? ~0ULL : ((1ULL << bits) - 1);
  fb_string_hash_kernel<<<grid_for(dev, n), kThreads, 0, (cudaStream_t)stream>>>(n, offsets, data, valid, mask, out);
  FB_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int fb_string_first_equal(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                                     const uint8_t* valid, const uint64_t* sorted_hash, const int64_t* sorted_idx,
                                     int64_t* canon) {
  FB_CHECK(n >= 0, "n < 0");
  if (n == 0) return 0;
  FB_CHECK(offsets != nullptr && data != nullptr && sorted_hash != nullptr && sorted_idx != nullptr &&
               canon != nullptr, "NULL argument");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  fb_string_first_equal_kernel<<<grid_for(dev, n), kThreads, 0, (cudaStream_t)stream>>>(
      n, offsets, data, valid, sorted_hash, sorted_idx, canon);
  FB_CUDA(cudaGetLastError());
  return 0;
}
