// The layout of the aligned power-of-two block tree of fb_window_tree / fb_window_bounded (fb_window.cu), shared
// with the kernels that read it (the range join walk in fb_join.cu).  Level l >= 1 holds nodes m < nrows >> l,
// node m covering rows [m 2^l, (m + 1) 2^l); level 0 is the input.  Level l starts at node off[l] of a column's
// `total` nodes.
#pragma once
#include <stdint.h>
#include <string.h>

constexpr int kTreeMaxLevels = 64;

struct TreeLevels {
  int64_t off[kTreeMaxLevels];
  int64_t total;  // nodes of levels >= 1 per column
  int levels;     // highest level with a node
};

inline TreeLevels tree_levels(int64_t nrows) {
  TreeLevels L;
  memset(&L, 0, sizeof(L));
  int64_t acc = 0;
  for (int l = 1; l < kTreeMaxLevels && (nrows >> l) > 0; ++l) {
    L.off[l] = acc;
    acc += nrows >> l;
    L.levels = l;
  }
  L.total = acc;
  return L;
}
