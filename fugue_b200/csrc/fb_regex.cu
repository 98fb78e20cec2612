// K15 regular expressions for sm_90a, evaluated once per dictionary entry (include/fugue_b200.h).
//
// The host compiles a pattern into positions (instructions that consume one code point) and closures: for each
// point a match can be at, the positions the empty-width part of the program reaches from it, in leftmost-first
// priority order, with the capture slots set on the way.  Assertions are decided when the closure is built
// (^ and \A hold only at byte 0, $ and \z only at the end), so a closure has two variants, "at the end" or not.
//
// fb_regex_match runs a bit-parallel Thompson machine: the live positions are one 64-bit word, and one code
// point ORs the closures of the live positions that accept it.  fb_regex_transform runs a Pike VM over the same
// closures: a list of threads in priority order, at most one per position, each with the slots the call needs.
// Both are one thread per entry, grid-stride; the thread lists are a fixed frame of the transform kernel, so the
// stack does not depend on the entry length.  fb_debug_regex_host runs the same per-entry code on the CPU.
#include "fb_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMatch = FB_REGEX_MAX_STATES;     // the match target of a closure entry
constexpr int kStart = FB_REGEX_MAX_STATES;     // closure row: a match starting away from byte 0
constexpr int kStartAt0 = FB_REGEX_MAX_STATES + 1;

FB_HD int ctz64(uint64_t x) {
#ifdef __CUDA_ARCH__
  return __ffsll((long long)x) - 1;
#else
  return __builtin_ctzll(x);
#endif
}

FB_HD int closure_id(int row, bool at_end) { return 2 * row + (at_end ? 1 : 0); }

// the code point at byte i of s[0, len) and the byte after it; a byte that does not start a well-formed
// sequence is one code point of its own (U+FFFD, which no ASCII-only class accepts)
FB_HD uint32_t next_cp(const uint8_t* s, int64_t len, int64_t i, int64_t* j) {
  const uint8_t b = s[i];
  if (b < 0x80) {
    *j = i + 1;
    return b;
  }
  const int k = b >= 0xF0 ? 4 : (b >= 0xE0 ? 3 : (b >= 0xC0 ? 2 : 0));
  bool ok = k > 0 && i + k <= len;
  uint32_t c = k == 4 ? (b & 0x07) : (k == 3 ? (b & 0x0F) : (b & 0x1F));
  for (int q = 1; ok && q < k; ++q) {
    ok = (s[i + q] & 0xC0) == 0x80;
    c = (c << 6) | (s[i + q] & 0x3F);
  }
  *j = ok ? i + k : i + 1;
  return ok ? c : 0xFFFD;
}

// the positions that accept code point c
FB_HD uint64_t accepts(const fb_regex_program& P, const uint64_t* ascii, uint32_t c) {
  if (c < 128) return ascii[c];
  int lo = 0, hi = P.nranges;  // the last range whose start is <= c
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (P.range_lo[mid] <= c) lo = mid; else hi = mid;
  }
  return P.nranges > 0 ? P.range_mask[lo] : 0;
}

// REGEXP_MATCHES over s[0, len): the Thompson machine; ascii / cl_mask / cl_accept may be shared-memory copies
FB_HD bool search(const fb_regex_program& P, const uint64_t* ascii, const uint64_t* cl_mask, const uint8_t* cl_accept,
                  const uint8_t* s, int64_t len) {
  int c0 = closure_id(kStartAt0, len == 0);
  if (cl_accept[c0]) return true;
  uint64_t live = cl_mask[c0];
  for (int64_t i = 0; i < len;) {
    int64_t j;
    const uint32_t c = next_cp(s, len, i, &j);
    const bool end = j == len;
    uint64_t step = live & accepts(P, ascii, c);
    const int cs = closure_id(kStart, end);
    uint64_t next = cl_mask[cs];
    bool acc = cl_accept[cs] != 0;
    while (step) {
      const int p = ctz64(step);
      step &= step - 1;
      next |= cl_mask[closure_id(p, end)];
      acc |= cl_accept[closure_id(p, end)] != 0;
    }
    if (acc) return true;
    live = next;
    if (live == 0 && !P.restart) return false;
    i = j;
  }
  return false;
}

// two lists of Pike VM threads (the current and the next code point), each in priority order, at most one
// thread per position and one at the match
template <int kSlots>
struct Threads {
  uint8_t pos[2][FB_REGEX_MAX_STATES + 1];
  int32_t slot[2][FB_REGEX_MAX_STATES + 1][kSlots];
};

// appends to list b the closure's entries that are not on it yet (on / on_match), with the slots it sets at byte
// `at`; the other slots come from thread t of the other list (t < 0: unset)
template <int kSlots>
FB_HD void add(const fb_regex_program& P, Threads<kSlots>& L, int b, int& n, uint64_t& on, bool& on_match, int c,
               int t, int32_t at) {
  for (int e = P.cl_off[c]; e < P.cl_off[c + 1]; ++e) {
    const int x = P.ent_target[e];
    if (x == kMatch) {
      if (on_match) continue;
      on_match = true;
    } else {
      if ((on >> x) & 1) continue;
      on |= 1ULL << x;
    }
    const int save = P.ent_save[e];
    L.pos[b][n] = (uint8_t)x;
    for (int q = 0; q < P.nslots; ++q)
      L.slot[b][n][q] = ((save >> q) & 1) ? at : (t >= 0 ? L.slot[b ^ 1][t][q] : -1);
    ++n;
  }
}

// the leftmost-first match in s[0, len) that starts at byte `from` or later; its slots go to m
template <int kSlots>
FB_HD bool pike(const fb_regex_program& P, const uint8_t* s, int64_t len, int64_t from, Threads<kSlots>& L,
                int32_t* m) {
  int b = 0, n = 0;
  uint64_t on = 0;
  bool on_match = false, found = false;
  add(P, L, b, n, on, on_match, closure_id(from == 0 ? kStartAt0 : kStart, from == len), -1, (int32_t)from);
  for (int64_t i = from;;) {
    if (i == len) {
      for (int t = 0; t < n; ++t) {
        if (L.pos[b][t] == kMatch) {
          for (int q = 0; q < P.nslots; ++q) m[q] = L.slot[b][t][q];
          return true;
        }
      }
      return found;
    }
    int64_t j;
    const uint32_t c = next_cp(s, len, i, &j);
    const bool end = j == len;
    const uint64_t acc = accepts(P, P.ascii, c);
    int nn = 0;
    uint64_t non = 0;
    bool nmatch = false;
    for (int t = 0; t < n; ++t) {
      const int p = L.pos[b][t];
      if (p == kMatch) {  // every thread after this one has a lower priority
        for (int q = 0; q < P.nslots; ++q) m[q] = L.slot[b][t][q];
        found = true;
        break;
      }
      if ((acc >> p) & 1) add(P, L, b ^ 1, nn, non, nmatch, closure_id(p, end), t, (int32_t)j);
    }
    if (!found) add(P, L, b ^ 1, nn, non, nmatch, closure_id(kStart, end), -1, (int32_t)j);
    b ^= 1;
    n = nn;
    on = non;
    on_match = nmatch;
    i = j;
    if (n == 0 && (found || !P.restart)) return found;
  }
}

// counts the output bytes; the writing emitter also stores them
template <bool kWrite>
struct Emit {
  uint8_t* out;
  int64_t n = 0;
  FB_HD void put(uint8_t b) {
    if (kWrite) out[n] = b;
    ++n;
  }
  FB_HD void put(const uint8_t* p, int64_t k) {
    if (kWrite)
      for (int64_t q = 0; q < k; ++q) out[n + q] = p[q];
    n += k;
  }
};

template <typename E>
FB_HD void rewrite(E& e, const fb_regex_program& P, const uint8_t* s, const int32_t* m) {
  for (int t = 0; t < P.nrewrite; ++t) {
    const int tk = P.rewrite[t];
    if (tk < FB_REGEX_GROUP) {
      e.put((uint8_t)tk);
    } else {
      const int k = tk - FB_REGEX_GROUP;
      if (m[2 * k] >= 0 && m[2 * k + 1] >= 0) e.put(s + m[2 * k], m[2 * k + 1] - m[2 * k]);
    }
  }
}

// the result of one entry into e (EXTRACT / REPLACE / REPLACE_ALL); pair 0 of the slots is the match
template <int kSlots, typename E>
FB_HD void transform(E& e, const fb_regex_program& P, const uint8_t* s, int64_t len, Threads<kSlots>& L) {
  int32_t m[kSlots];
  if (P.op == FB_REGEX_EXTRACT) {
    if (pike<kSlots>(P, s, len, 0, L, m)) {
      const int k = P.group_pair;
      if (m[2 * k] >= 0 && m[2 * k + 1] >= 0) e.put(s + m[2 * k], m[2 * k + 1] - m[2 * k]);
    }
    return;
  }
  int64_t p = 0, last_end = -1;
  while (p <= len) {
    if (!pike<kSlots>(P, s, len, p, L, m)) break;
    if (m[0] == last_end && m[1] == m[0]) {  // an empty match right after the previous match: skip a code point
      if (p == len) break;
      int64_t j;
      next_cp(s, len, p, &j);
      e.put(s + p, j - p);
      p = j;
      continue;
    }
    e.put(s + p, m[0] - p);
    rewrite(e, P, s, m);
    p = last_end = m[1];
    if (P.op == FB_REGEX_REPLACE) break;
  }
  if (p < len) e.put(s + p, len - p);
}

__global__ void __launch_bounds__(kThreads)
fb_regex_match_kernel(const fb_regex_program* __restrict__ P, int64_t n, const int64_t* __restrict__ offsets,
                      const uint8_t* __restrict__ data, const uint8_t* __restrict__ valid, uint8_t* __restrict__ out,
                      uint8_t* __restrict__ out_valid) {
  __shared__ uint64_t s_ascii[128];
  __shared__ uint64_t s_mask[FB_REGEX_MAX_CLOSURES];
  __shared__ uint8_t s_accept[FB_REGEX_MAX_CLOSURES];
  for (int q = threadIdx.x; q < 128; q += kThreads) s_ascii[q] = P->ascii[q];
  for (int q = threadIdx.x; q < FB_REGEX_MAX_CLOSURES; q += kThreads) {
    s_mask[q] = P->cl_mask[q];
    s_accept[q] = P->cl_accept[q];
  }
  __syncthreads();
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const bool ok = valid == nullptr || valid[i] != 0;
    const int64_t a = offsets[i];
    out[i] = ok && search(*P, s_ascii, s_mask, s_accept, data + a, offsets[i + 1] - a) ? 1 : 0;
    out_valid[i] = ok ? 1 : 0;
  }
}

template <int kSlots>
__global__ void __launch_bounds__(kThreads)
fb_regex_transform_kernel(const fb_regex_program* __restrict__ P, int64_t n, const int64_t* __restrict__ offsets,
                          const uint8_t* __restrict__ data, const uint8_t* __restrict__ valid,
                          int64_t* __restrict__ out_len, uint8_t* __restrict__ out_valid,
                          const int64_t* __restrict__ out_offsets, uint8_t* __restrict__ out_data) {
  Threads<kSlots> L;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const bool ok = valid == nullptr || valid[i] != 0;
    const int64_t a = offsets[i];
    if (out_data == nullptr) {
      Emit<false> e{nullptr};
      if (ok) transform<kSlots>(e, *P, data + a, offsets[i + 1] - a, L);
      out_len[i] = ok ? e.n : 0;
      out_valid[i] = ok ? 1 : 0;
    } else if (ok) {
      Emit<true> e{out_data + out_offsets[i]};
      transform<kSlots>(e, *P, data + a, offsets[i + 1] - a, L);
    }
  }
}

unsigned grid_for(int dev, int64_t n) {
  const int64_t blocks = (n + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)fb_sm_count(dev) * 8;
  return (unsigned)(blocks < cap ? blocks : cap);
}

// the checks every entry point makes on a program before any kernel reads it
int check_program(const fb_regex_program* P, bool match) {
  FB_CHECK(P != nullptr, "NULL program");
  FB_CHECK(P->npos >= 0 && P->npos <= FB_REGEX_MAX_STATES, "npos=%d out of range [0,%d]", P->npos,
           FB_REGEX_MAX_STATES);
  FB_CHECK(P->nranges >= 0 && P->nranges <= FB_REGEX_MAX_RANGES, "nranges=%d out of range [0,%d]", P->nranges,
           FB_REGEX_MAX_RANGES);
  FB_CHECK(P->nranges == 0 || P->range_lo[0] == 128, "range_lo[0] must be 128");
  for (int r = 1; r < P->nranges; ++r)
    FB_CHECK(P->range_lo[r] > P->range_lo[r - 1] && P->range_lo[r] <= 0x10FFFF, "range_lo not increasing at %d", r);
  FB_CHECK(P->cl_off[0] == 0, "cl_off[0] != 0");
  for (int c = 0; c < FB_REGEX_MAX_CLOSURES; ++c)
    FB_CHECK(P->cl_off[c + 1] >= P->cl_off[c] && P->cl_off[c + 1] <= FB_REGEX_MAX_ENTRIES, "cl_off bad at %d", c);
  for (int e = 0; e < P->cl_off[FB_REGEX_MAX_CLOSURES]; ++e)
    FB_CHECK(P->ent_target[e] < P->npos || P->ent_target[e] == kMatch, "entry %d: target %d", e, P->ent_target[e]);
  if (match) {
    FB_CHECK(P->op == FB_REGEX_MATCH, "op %d is not FB_REGEX_MATCH", P->op);
    return 0;
  }
  FB_CHECK(P->op >= FB_REGEX_EXTRACT && P->op <= FB_REGEX_REPLACE_ALL, "unknown op %d", P->op);
  FB_CHECK(P->nslots >= 2 && P->nslots <= FB_REGEX_MAX_SLOTS && P->nslots % 2 == 0, "nslots=%d out of range",
           P->nslots);
  FB_CHECK(P->op != FB_REGEX_EXTRACT || (P->group_pair >= 0 && 2 * P->group_pair < P->nslots),
           "group_pair=%d out of range", P->group_pair);
  FB_CHECK(P->nrewrite >= 0 && P->nrewrite <= FB_REGEX_MAX_REWRITE, "nrewrite=%d out of range", P->nrewrite);
  for (int t = 0; t < P->nrewrite; ++t)
    FB_CHECK(P->rewrite[t] >= 0 && (P->rewrite[t] < FB_REGEX_GROUP || 2 * (P->rewrite[t] - FB_REGEX_GROUP) < P->nslots),
             "rewrite token %d: %d", t, (int)P->rewrite[t]);
  return 0;
}

}  // namespace

extern "C" int fb_regex_match(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                              const uint8_t* valid, const fb_regex_program* prog, const fb_regex_program* dprog,
                              uint8_t* out, uint8_t* out_valid) {
  FB_CHECK(n >= 0, "n < 0");
  if (check_program(prog, true) != 0) return 1;
  if (n == 0) return 0;
  FB_CHECK(offsets != nullptr && data != nullptr && dprog != nullptr && out != nullptr && out_valid != nullptr,
           "NULL argument");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  fb_regex_match_kernel<<<grid_for(dev, n), kThreads, 0, (cudaStream_t)stream>>>(dprog, n, offsets, data, valid, out,
                                                                                 out_valid);
  FB_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int fb_regex_transform(int dev, void* stream, int64_t n, const int64_t* offsets, const uint8_t* data,
                                  const uint8_t* valid, const fb_regex_program* prog, const fb_regex_program* dprog,
                                  int64_t* out_len, uint8_t* out_valid, const int64_t* out_offsets,
                                  uint8_t* out_data) {
  FB_CHECK(n >= 0, "n < 0");
  if (check_program(prog, false) != 0) return 1;
  if (n == 0) return 0;
  FB_CHECK(offsets != nullptr && data != nullptr && dprog != nullptr, "NULL argument");
  FB_CHECK(out_data != nullptr ? out_offsets != nullptr : (out_len != nullptr && out_valid != nullptr),
           "NULL output");
  FbDeviceGuard guard(dev);
  FB_CHECK(guard.ok, "cannot select device %d", dev);
  const unsigned grid = grid_for(dev, n);
  if (prog->nslots <= 2)
    fb_regex_transform_kernel<2><<<grid, kThreads, 0, (cudaStream_t)stream>>>(dprog, n, offsets, data, valid,
                                                                               out_len, out_valid, out_offsets, out_data);
  else
    fb_regex_transform_kernel<FB_REGEX_MAX_SLOTS><<<grid, kThreads, 0, (cudaStream_t)stream>>>(
        dprog, n, offsets, data, valid, out_len, out_valid, out_offsets, out_data);
  FB_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int fb_debug_regex_host(int64_t n, const int64_t* offsets, const uint8_t* data, const uint8_t* valid,
                                   const fb_regex_program* prog, int64_t* out_len, uint8_t* out_valid,
                                   const int64_t* out_offsets, uint8_t* out_data) {
  FB_CHECK(n >= 0, "n < 0");
  const bool match = prog != nullptr && prog->op == FB_REGEX_MATCH;
  if (check_program(prog, match) != 0) return 1;
  if (n == 0) return 0;
  FB_CHECK(offsets != nullptr && data != nullptr, "NULL argument");
  FB_CHECK(out_data != nullptr ? out_offsets != nullptr : (out_len != nullptr && out_valid != nullptr),
           "NULL output");
  Threads<FB_REGEX_MAX_SLOTS> L;
  for (int64_t i = 0; i < n; ++i) {
    const bool ok = valid == nullptr || valid[i] != 0;
    const uint8_t* s = data + offsets[i];
    const int64_t len = offsets[i + 1] - offsets[i];
    if (match) {
      out_len[i] = ok && search(*prog, prog->ascii, prog->cl_mask, prog->cl_accept, s, len) ? 1 : 0;
      out_valid[i] = ok ? 1 : 0;
    } else if (out_data == nullptr) {
      Emit<false> e{nullptr};
      if (ok) transform<FB_REGEX_MAX_SLOTS>(e, *prog, s, len, L);
      out_len[i] = ok ? e.n : 0;
      out_valid[i] = ok ? 1 : 0;
    } else if (ok) {
      Emit<true> e{out_data + out_offsets[i]};
      transform<FB_REGEX_MAX_SLOTS>(e, *prog, s, len, L);
    }
  }
  return 0;
}
