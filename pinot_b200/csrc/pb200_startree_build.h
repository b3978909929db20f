// pb200_startree_build.h -- device-side star-tree build (pb200_startree_build.cu), called by pb200h_startree_build.
#pragma once
#include <cstdint>
#include <vector>

#include "pb200_internal.h"

namespace pb200 {

// One tree to build over the columns of `seg` (column ids of the device segment).  The caller has checked the names,
// the kinds of the columns and the functions (host/star_tree.cpp).
struct StarBuildSpec {
  std::vector<int> dim_cols;        // split order
  std::vector<char> skip_star;      // per dimension: skipStarNodeCreationForDimensions
  std::vector<int> metric_fn;       // PB200_AGG_COUNT / SUM / MIN / MAX
  std::vector<int> metric_col;      // -1 for COUNT
  int max_leaf_records = 10000;
};

enum { STAR_PHASE_BASE = 0, STAR_PHASE_CONSTRUCT = 1, STAR_PHASE_AGGREGATE = 2, STAR_PHASE_ENCODE = 3, STAR_PHASES = 4 };

struct StarBuildResult {
  std::vector<int32_t> nodes;       // 7 ints per node, breadth first: dim, value, start, end, agg, first child, last child
  long long num_base_docs = 0;
  pb200_segment* docs = nullptr;    // the star docs: dimensions (dictIds of the base dictionaries), then the metrics
                                    // (count__* LONG, the others DOUBLE, dictionary encoded), then hidden limb columns
  // Per metric: -1, or for SUM over an INT column the first of three raw INT columns of `docs` that hold each star doc's
  // exact sum x as limbs, x = l2 * 2^42 + l1 * 2^21 + l0 (l0, l1 in [0, 2^21)).  A query's limb sums stay below 2^52
  // in magnitude for any number of star docs, so they come back from the scan exact in double; the DOUBLE sum__ column
  // holds x rounded, and a sum of those would round once per star doc.
  std::vector<int> limb_col;
  double ms[STAR_PHASES] = {};
};

// PB200_OK, or PB200_E_UNSUPPORTED / _NOMEM / _CUDA with the message set; nothing is returned on failure
int startree_build(pb200_ctx* ctx, const pb200_segment* seg, const StarBuildSpec& spec, StarBuildResult* out);

}  // namespace pb200
