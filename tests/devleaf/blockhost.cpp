// blockhost.cpp -- TEST HELPER ONLY.  The compaction primitives of block.h built with g++ as a one-thread CTA (tid = 0,
// nt = 1, barriers are no-ops): the host twin of blockleaf.cu's k_inlidxs.  tests/devleaf/blk.py loads it with ctypes.
#include <string.h>
#include "../../pydegensac_b200/csrc/block.h"

using namespace dg;

// blk_inlidxs (two = 0: two calls) or blk_inlidxs2 (two = 1): lists, J[2], I[3] (I[2] = blk_count_lt(thA))
extern "C" void hb_blk_inlidxs(const double* err, int N, double thA, double thB, int two, int* listA, int* listB,
                               double* J, int* I) {
  static BlockScratch sc;
  Ctx c;
  memset(&c, 0, sizeof(c));
  c.nt = 1; c.nw = 1; c.N = N; c.sc = &sc;
  Score SA, SB;
  if (two) {
    blk_inlidxs2(c, err, thA, listA, &SA, thB, listB, &SB);
  } else {
    SA = blk_inlidxs(c, err, thA, listA);
    SB = blk_inlidxs(c, err, thB, listB);
  }
  J[0] = SA.J; J[1] = SB.J; I[0] = (int)SA.I; I[1] = (int)SB.I; I[2] = blk_count_lt(c, err, thA);
}
