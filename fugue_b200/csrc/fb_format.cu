// K14 number / bool / date / timestamp -> string casts for sm_90a (include/fugue_b200.h).  The format routines are
// fb_format.cuh; fb_debug_value_format_host runs the same routines on the CPU.
//
// One thread per value, grid-stride, in two launches like K12: the measure call counts each value's bytes, the host
// scans the counts into offsets, and the write call stores the bytes at them.
#include "fb_format.cuh"

namespace {

constexpr int kFormatThreads = 256;

__global__ void __launch_bounds__(kFormatThreads)
fb_value_format_kernel(int64_t n, const uint64_t* __restrict__ values, const uint8_t* __restrict__ valid, int kind,
                       int64_t* __restrict__ out_len, const int64_t* __restrict__ out_offsets,
                       uint8_t* __restrict__ out_data) {
  for (int64_t i = (int64_t)blockIdx.x * kFormatThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kFormatThreads) {
    const bool ok = valid == nullptr || valid[i] != 0;
    const uint64_t v = __ldg((const unsigned long long*)values + i);
    if (out_data == nullptr) {
      FbCount c;
      if (ok) fb_format_value(c, v, kind);
      out_len[i] = c.n;
    } else if (ok) {
      FbStore s{out_data + out_offsets[i]};
      fb_format_value(s, v, kind);
    }
  }
}

bool kind_ok(int kind) {
  return (kind >= FB_FMT_I64 && kind <= FB_FMT_DATE64) ||
         ((kind & ~(FB_FMT_TS_FRAC | 7)) == FB_FMT_TS && (kind & 7) >= FB_TU_S && (kind & 7) <= FB_TU_NS &&
          !((kind & FB_FMT_TS_FRAC) && (kind & 7) == FB_TU_S));
}

}  // namespace

extern "C" int fb_value_format(int dev, void* stream, int64_t n, const uint64_t* values, const uint8_t* valid,
                               int kind, int64_t* out_len, const int64_t* out_offsets, uint8_t* out_data) {
  FB_CHECK(n >= 0, "n < 0");
  FB_CHECK(kind_ok(kind), "unknown format kind %d", kind);
  if (n == 0) return 0;
  FB_CHECK(values != nullptr, "NULL argument");
  FB_CHECK(out_data != nullptr ? out_offsets != nullptr : out_len != nullptr, "NULL argument");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  const int64_t blocks = (n + kFormatThreads - 1) / kFormatThreads, cap = (int64_t)fb_sm_count(dev) * 8;
  fb_value_format_kernel<<<(unsigned)(blocks < cap ? blocks : cap), kFormatThreads, 0, (cudaStream_t)stream>>>(
      n, values, valid, kind, out_len, out_offsets, out_data);
  FB_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int fb_debug_value_format_host(int64_t n, const uint64_t* values, const uint8_t* valid, int kind,
                                          int64_t* out_len, const int64_t* out_offsets, uint8_t* out_data) {
  FB_CHECK(n >= 0, "n < 0");
  FB_CHECK(kind_ok(kind), "unknown format kind %d", kind);
  FB_CHECK(n == 0 || (values != nullptr && (out_data != nullptr ? out_offsets != nullptr : out_len != nullptr)),
           "NULL argument");
  for (int64_t i = 0; i < n; ++i) {
    const bool ok = valid == nullptr || valid[i] != 0;
    if (out_data == nullptr) {
      FbCount c;
      if (ok) fb_format_value(c, values[i], kind);
      out_len[i] = c.n;
    } else if (ok) {
      FbStore s{out_data + out_offsets[i]};
      fb_format_value(s, values[i], kind);
    }
  }
  return 0;
}
