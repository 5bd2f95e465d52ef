// Device half of the reference-ordered ("exact") selection order (a16): the reference
// builds the candidate list in block-raster order and std::sort()s it by key
// (g/processor.cc:636-678); where equal keys of different blocks decide the walk, the
// arrangement introsort leaves behind has to be reproduced (exact_sort.h).  Replaying
// libstdc++'s introsort costs one pass over the whole list per partition level, which
// for a 4K image is most of an iteration's wall time on the host.  These functors move
// the list and the partition passes over large ranges onto the device:
//   OrderRefCount / OrderRefBuild   the list in the reference's own order
//   OrderPivot                      std::__move_median_to_first
//   OrderPartFlags .. OrderPartSwap std::__unguarded_partition, in parallel: the
//       sequential scan swaps the k-th element >= pivot from the left with the k-th
//       element <= pivot from the right while they have not crossed, which is what the
//       two rank lists reproduce.
// Ranges below a threshold go back to the host replay.  Checked against the host replay on
// the CPU port and on the GPU (tools/check_device_order.py); GB200_DEVICE_ORDER=0 disables.
#pragma once
#include "hd.h"
#include "kernels.h"

namespace gb200 {

struct OrderItem {  // layout of std::pair<int, float>
  int block;
  float key;
};

struct OrderRefCount {  // 1D over blocks: entries of block b in the order (g/processor.cc:636-663)
  const int* last_index;
  const int* cand_count;
  const float* weight;
  int direction;
  unsigned int* count;
  GB_HD void operator()(int b) const {
    const int li = last_index[b], nc = cand_count[b];
    unsigned int n = 0;
    if (weight[b] != 0) n = direction > 0 ? (li < nc ? nc - li : 0) : (li > 0 ? li : 0);
    count[b] = n;
  }
};

struct OrderRefBuild {  // 1D over candidate entries
  OrderKeyCommon c;
  const unsigned int* offset;  // exclusive scan of OrderRefCount
  OrderItem* out;
  GB_HD void operator()(int e) const {
    int b;
    float val;
    if (!c.key(e, &b, &val)) return;
    const int slot = c.entry_slot[e], li = c.last_index[b];
    const unsigned int pos = offset[b] + static_cast<unsigned int>(c.direction > 0 ? slot - li : li - 1 - slot);
    out[pos].block = b;
    out[pos].key = val;
  }
};

struct OrderPivot {  // one thread: median of a[f+1], a[mid], a[l-1] swapped into a[f]
  OrderItem* a;
  long long f, l;
  GB_HD void operator()(int) const {
    const long long ia = f + 1, ib = f + (l - f) / 2, ic = l - 1;
    const float ka = a[ia].key, kb = a[ib].key, kc = a[ic].key;
    long long pick;
    if (ka < kb) {
      pick = kb < kc ? ib : (ka < kc ? ic : ia);
    } else if (ka < kc) {
      pick = ia;
    } else {
      pick = kb < kc ? ic : ib;
    }
    const OrderItem t = a[f];
    a[f] = a[pick];
    a[pick] = t;
  }
};

// Range R = [f+1, l), m = l - f - 1 elements, pivot a[f].  fl[t] = element t of R is not
// below the pivot; fr[u] = element m-1-u of R is not above it (reversed, so that an
// exclusive scan of fr ranks the elements from the right).
struct OrderPartFlags {
  const OrderItem* a;
  long long f;
  int m;
  unsigned int* fl;
  unsigned int* fr;
  GB_HD void operator()(int t) const {
    const float p = a[f].key, k = a[f + 1 + t].key;
    fl[t] = !(k < p) ? 1u : 0u;
    fr[m - 1 - t] = !(p < k) ? 1u : 0u;
  }
};

// Rank lists and the number of swaps.  An element of the left list with rank k is swapped
// iff at least k+1 right-list elements lie beyond it.
struct OrderPartLists {
  const unsigned int* fl;
  const unsigned int* sl;  // exclusive scan of fl
  const unsigned int* fr;
  const unsigned int* sr;  // exclusive scan of fr
  int m;
  int* llist;              // position (index t in R) of the k-th left element
  int* rlist;              // position of the k-th right element
  unsigned int* num_swaps;
  GB_HD void operator()(int t) const {
    if (fl[t]) {
      llist[sl[t]] = t;
      if (sr[m - 1 - t] >= sl[t] + 1u) hd_atomic_add(num_swaps, 1u);
    }
    const int u = m - 1 - t;
    if (fr[u]) rlist[sr[u]] = t;
  }
};

struct OrderPartSwap {  // 1D over the swaps
  OrderItem* a;
  long long f;
  const int* llist;
  const int* rlist;
  GB_HD void operator()(int k) const {
    const long long i = f + 1 + llist[k], j = f + 1 + rlist[k];
    const OrderItem t = a[i];
    a[i] = a[j];
    a[j] = t;
  }
};

// One thread: where the sequential scan's `lo` ends up (the cut), as an index into a[].
struct OrderPartCut {
  long long f;
  const int* llist;
  const int* rlist;
  const unsigned int* num_swaps;
  unsigned int total_l;
  long long* cut;
  GB_HD void operator()(int) const {
    const unsigned int k = *num_swaps;
    long long lo = -1;
    if (k < total_l) lo = llist[k];
    if (k >= 1 && (lo < 0 || rlist[k - 1] < lo)) lo = rlist[k - 1];  // the element swapped there stops the scan first
    *cut = f + 1 + lo;
  }
};

}  // namespace gb200
