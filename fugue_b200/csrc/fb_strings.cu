// K11 string functions for sm_90a, evaluated once per dictionary entry (include/fugue_b200.h).
//
// String columns are dictionary encoded: int32 codes per row, one Arrow string array per column as the
// dictionary.  LIKE and LENGTH depend on the string alone, so they run over the dictionary's entries -
// usually far fewer than the rows - and the expression evaluator (K8, FB_X_LOOKUP) then maps every row's
// code to its entry's result inside the same one-pass program as the rest of the SELECT list.
//
// One thread per entry, grid-stride.  The pattern (at most FB_LIKE_MAX_TOKENS tokens) is a kernel
// parameter, so every thread reads it from the constant bank.
#include "fb_common.cuh"

namespace {

constexpr int kStrThreads = 256;

struct LikeProgram {
  int32_t ntok;
  int16_t tok[FB_LIKE_MAX_TOKENS];
};
static_assert(sizeof(LikeProgram) <= 4000, "pattern must fit the kernel parameter space");

__device__ __forceinline__ bool is_cont(uint8_t b) { return (b & 0xC0) == 0x80; }

// byte length of the code point whose lead byte is b (a stray continuation byte counts as one)
__device__ __forceinline__ int cp_len(uint8_t b) {
  return b < 0xC0 ? 1 : (b < 0xE0 ? 2 : (b < 0xF0 ? 3 : 4));
}

// match tokens [t0, t1) at byte p of s[0, len); returns the end byte or -1
__device__ int64_t match_at(const LikeProgram& P, int t0, int t1, const uint8_t* __restrict__ s, int64_t len,
                            int64_t p) {
  for (int t = t0; t < t1; ++t) {
    if (p >= len) return -1;
    const int tk = P.tok[t];
    const uint8_t c = s[p];
    if (tk == FB_LIKE_ONE) {
      p += cp_len(c);
      if (p > len) return -1;
    } else {
      if (c != (uint8_t)tk) return -1;
      ++p;
    }
  }
  return p;
}

__device__ bool like_entry(const LikeProgram& P, const uint8_t* __restrict__ s, int64_t len) {
  int seg_end = 0;  // first segment: tokens [0, seg_end)
  while (seg_end < P.ntok && P.tok[seg_end] != FB_LIKE_ANY) ++seg_end;
  if (seg_end == P.ntok) return match_at(P, 0, P.ntok, s, len, 0) == len;  // no '%': the whole string
  int64_t p = match_at(P, 0, seg_end, s, len, 0);                         // anchored at the start
  if (p < 0) return false;
  int t0 = seg_end + 1;
  for (;;) {
    int t1 = t0;
    while (t1 < P.ntok && P.tok[t1] != FB_LIKE_ANY) ++t1;
    if (t1 == P.ntok) break;  // [t0, ntok) is the last segment
    // a middle segment: its leftmost match at a code-point boundary at or after p
    int64_t end = -1;
    for (int64_t q = p; q < len; ++q) {
      if (is_cont(s[q])) continue;
      end = match_at(P, t0, t1, s, len, q);
      if (end >= 0) break;
    }
    if (end < 0) return false;
    p = end;
    t0 = t1 + 1;
  }
  // the last segment, anchored at the end: it covers as many code points as it has tokens that start one
  int cps = 0;
  for (int t = t0; t < P.ntok; ++t) cps += P.tok[t] == FB_LIKE_ONE || !is_cont((uint8_t)P.tok[t]);
  int64_t q = len;
  for (int k = 0; k < cps; ++k) {
    do {
      if (q == p) return false;  // not enough code points after the previous segment
      --q;
    } while (is_cont(s[q]));
  }
  return match_at(P, t0, P.ntok, s, len, q) == len;
}

__global__ void __launch_bounds__(kStrThreads)
fb_string_like_kernel(const __grid_constant__ LikeProgram P, int64_t n, const int64_t* __restrict__ offsets,
                      const uint8_t* __restrict__ data, const uint8_t* __restrict__ valid,
                      uint8_t* __restrict__ out, uint8_t* __restrict__ out_valid) {
  for (int64_t i = (int64_t)blockIdx.x * kStrThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kStrThreads) {
    const bool ok = valid == nullptr || valid[i] != 0;
    const int64_t a = offsets[i];
    out[i] = ok && like_entry(P, data + a, offsets[i + 1] - a) ? 1 : 0;
    out_valid[i] = ok ? 1 : 0;
  }
}

__global__ void __launch_bounds__(kStrThreads)
fb_string_length_kernel(int64_t n, const int64_t* __restrict__ offsets, const uint8_t* __restrict__ data,
                        const uint8_t* __restrict__ valid, int64_t* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * kStrThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kStrThreads) {
    int64_t cps = 0;
    if (valid == nullptr || valid[i] != 0) {
      const int64_t a = offsets[i], b = offsets[i + 1];
      for (int64_t p = a; p < b; ++p) cps += !is_cont(data[p]);
    }
    out[i] = cps;
  }
}

unsigned str_grid(int dev, int64_t n) {
  const int64_t blocks = (n + kStrThreads - 1) / kStrThreads;
  const int64_t cap = (int64_t)fb_sm_count(dev) * 8;
  return (unsigned)(blocks < cap ? blocks : cap);
}

}  // namespace

extern "C" int fb_string_length(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                                const uint8_t* valid, int64_t* out) {
  FB_CHECK(n >= 0, "n < 0");
  if (n == 0) return 0;
  FB_CHECK(offsets != nullptr && out != nullptr, "NULL argument");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  fb_string_length_kernel<<<str_grid(dev, n), kStrThreads, 0, (cudaStream_t)stream>>>(n, offsets, data, valid, out);
  FB_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int fb_string_like(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                              const uint8_t* valid, int ntokens, const int16_t* tokens, uint8_t* out,
                              uint8_t* out_valid) {
  FB_CHECK(n >= 0, "n < 0");
  FB_CHECK(ntokens >= 0 && ntokens <= FB_LIKE_MAX_TOKENS, "ntokens=%d out of range [0,%d]", ntokens,
           FB_LIKE_MAX_TOKENS);
  FB_CHECK(ntokens == 0 || tokens != nullptr, "NULL pattern");
  LikeProgram P;
  memset(&P, 0, sizeof(P));
  for (int t = 0; t < ntokens; ++t) {
    FB_CHECK(tokens[t] >= 0 && tokens[t] <= FB_LIKE_ANY, "token %d: unknown value %d", t, (int)tokens[t]);
    FB_CHECK(!(tokens[t] == FB_LIKE_ANY && t > 0 && tokens[t - 1] == FB_LIKE_ANY), "token %d: two '%%' in a row", t);
    P.tok[t] = tokens[t];
  }
  P.ntok = ntokens;
  if (n == 0) return 0;
  FB_CHECK(offsets != nullptr && out != nullptr && out_valid != nullptr, "NULL argument");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  fb_string_like_kernel<<<str_grid(dev, n), kStrThreads, 0, (cudaStream_t)stream>>>(P, n, offsets, data, valid, out,
                                                                                   out_valid);
  FB_CUDA(cudaGetLastError());
  return 0;
}
