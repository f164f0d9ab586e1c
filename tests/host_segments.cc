// host_segments.cc -- CPU check of the "fast" segmented warp reduction (seg_reduce_to): tba_segments.h's run_last_lane is the
// product's code; the two reductions are emulated lane by lane with the shuffle semantics of __shfl_down_sync (a lane whose
// source is out of range keeps its own value).
#include <cstdint>
#include "../theiasfm_b200/csrc/tba_segments.h"

extern "C" int host_run_last_lane(unsigned heads, int lane) { return tba::run_last_lane(heads, lane); }

// both reductions on one warp: keys[32], vals[32] -> out_key[32] (seg_reduce), out_fast[32] (seg_reduce_to)
extern "C" void host_seg_reduce_both(const int* keys, const double* vals, double* out_key, double* out_fast) {
  unsigned heads = 0;
  for (int l = 0; l < 32; ++l) if (l == 0 || keys[l - 1] != keys[l]) heads |= 1u << l;
  double a[32], b[32];
  for (int l = 0; l < 32; ++l) a[l] = b[l] = vals[l];
  for (int o = 1; o < 32; o <<= 1) {
    double na[32], nb[32];
    for (int l = 0; l < 32; ++l) {
      const double ova = l + o < 32 ? a[l + o] : a[l];
      const int ok = l + o < 32 ? keys[l + o] : keys[l];
      na[l] = (l + o < 32 && ok == keys[l]) ? a[l] + ova : a[l];
      const double ovb = l + o < 32 ? b[l + o] : b[l];
      nb[l] = (l + o <= tba::run_last_lane(heads, l)) ? b[l] + ovb : b[l];
    }
    for (int l = 0; l < 32; ++l) { a[l] = na[l]; b[l] = nb[l]; }
  }
  for (int l = 0; l < 32; ++l) { out_key[l] = a[l]; out_fast[l] = b[l]; }
}
