// K13 string -> number / bool / date / timestamp casts for sm_90a, evaluated once per dictionary entry
// (include/fugue_b200.h).  The parse routines are fb_strparse.cuh; fb_debug_string_parse_host runs the same
// routines on the CPU.
//
// One thread per entry, grid-stride, like the K11 functions: K8 then maps every row's code to its entry's value
// (FB_X_LOOKUP).  The smallest entry whose status is invalid or undecided is kept in one device word
// (atomicMin), so the host learns "every entry parsed" from one 8-byte read.
#include "fb_strparse.cuh"

namespace {

constexpr int kParseThreads = 256;

__global__ void __launch_bounds__(kParseThreads)
fb_string_parse_kernel(int64_t n, const int64_t* __restrict__ offsets, const uint8_t* __restrict__ data,
                       const uint8_t* __restrict__ valid, int target, uint64_t* __restrict__ out,
                       uint8_t* __restrict__ out_valid, uint8_t* __restrict__ status,
                       unsigned long long* __restrict__ first_bad) {
  unsigned long long bad = ~0ull;
  for (int64_t i = (int64_t)blockIdx.x * kParseThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kParseThreads) {
    uint64_t v = 0;
    uint8_t st = FB_PARSE_NULL;
    if (valid == nullptr || valid[i] != 0) {
      const int64_t a = offsets[i];
      st = fb_parse_entry(data + a, offsets[i + 1] - a, target, v);
    }
    out[i] = v;
    out_valid[i] = st == FB_PARSE_OK;
    status[i] = st;
    if (st >= FB_PARSE_INVALID && (unsigned long long)i < bad) bad = (unsigned long long)i;
  }
  if (bad != ~0ull) atomicMin(first_bad, bad);
}

bool target_ok(int target) {
  return (target >= FB_PARSE_I8 && target <= FB_PARSE_DATE64) ||
         ((target & ~(FB_PARSE_TS_ZONED | 7)) == FB_PARSE_TS && (target & 7) >= FB_TU_S && (target & 7) <= FB_TU_NS);
}

}  // namespace

extern "C" int fb_string_parse(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                               const uint8_t* valid, int target, uint64_t* out, uint8_t* out_valid, uint8_t* status,
                               uint64_t* first_bad) {
  FB_CHECK(n >= 0, "n < 0");
  FB_CHECK(target_ok(target), "unknown parse target %d", target);
  FB_CHECK(first_bad != nullptr, "NULL argument");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  FB_CUDA(cudaMemsetAsync(first_bad, 0xFF, sizeof(uint64_t), (cudaStream_t)stream));
  if (n == 0) return 0;
  FB_CHECK(offsets != nullptr && data != nullptr && out != nullptr && out_valid != nullptr && status != nullptr,
           "NULL argument");
  const int64_t blocks = (n + kParseThreads - 1) / kParseThreads, cap = (int64_t)fb_sm_count(dev) * 8;
  fb_string_parse_kernel<<<(unsigned)(blocks < cap ? blocks : cap), kParseThreads, 0, (cudaStream_t)stream>>>(
      n, offsets, data, valid, target, out, out_valid, status, (unsigned long long*)first_bad);
  FB_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int fb_debug_string_parse_host(int64_t n, const int64_t* offsets, const uint8_t* data,
                                          const uint8_t* valid, int target, uint64_t* out, uint8_t* out_valid,
                                          uint8_t* status) {
  FB_CHECK(n >= 0, "n < 0");
  FB_CHECK(target_ok(target), "unknown parse target %d", target);
  for (int64_t i = 0; i < n; ++i) {
    uint64_t v = 0;
    uint8_t st = FB_PARSE_NULL;
    if (valid == nullptr || valid[i] != 0) st = fb_parse_entry(data + offsets[i], offsets[i + 1] - offsets[i], target, v);
    out[i] = v;
    out_valid[i] = st == FB_PARSE_OK;
    status[i] = st;
  }
  return 0;
}
