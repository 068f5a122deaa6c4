/* TEST INFRASTRUCTURE ONLY (oracle/). Not part of the product path.
 *
 * k-nearest-neighbour match, bruce_slam/src/bruce_slam/cpp/pcl.cpp:161-174 with knn > 1: libpointmatcher's
 * KDTreeMatcher{knn, maxDist}, i.e. libnabo's exact k-NN search with a radius.  libnabo is not vendored or installed
 * here (parity unpinned, as for orc_match in cloud_ref.c), so this restates the rule by brute force, with the
 * conventions of orc_match_brute:
 *   distance   squared float32 dx*dx + dy*dy, each product and the sum rounded separately (built with
 *              -ffp-contract=off); a reference point counts when dist <= maxDist^2 (libnabo `dist <= maxRadius2`);
 *              a distance of +inf or NaN never counts
 *   order      ascending distance, ties -> lower reference index (libnabo's own tie order follows its tree
 *              traversal: a modelling choice)
 *   layout     ids / dists [knn][n_in]: row j holds every query's j-th neighbour; slots with no neighbour left hold
 *              id -1, dist +inf (also when knn exceeds the reference size)
 * Row 0 equals orc_match_brute's result, and rows 0 .. k-1 do not depend on knn >= k.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

void orc_match_knn(const float *ref, int n_ref, const float *in, int n_in, int knn, float max_dist, int32_t *ids,
                   float *dists) {
  const float max_d2 = max_dist * max_dist;
  if (knn < 1) return;
  for (int i = 0; i < n_in; ++i) {
    int k = 0;
    for (int j = 0; j < n_ref; ++j) {
      const float dx = in[2 * i] - ref[2 * j], dy = in[2 * i + 1] - ref[2 * j + 1];
      const float d2 = dx * dx + dy * dy;
      if (!(d2 <= max_d2) || !(d2 < INFINITY)) continue;
      /* j ascending: an equal distance never moves ahead of a listed (lower) index */
      if (k == knn && !(d2 < dists[(size_t)(knn - 1) * n_in + i])) continue;
      int at = k < knn ? k++ : knn - 1;
      while (at > 0 && d2 < dists[(size_t)(at - 1) * n_in + i]) {
        dists[(size_t)at * n_in + i] = dists[(size_t)(at - 1) * n_in + i];
        ids[(size_t)at * n_in + i] = ids[(size_t)(at - 1) * n_in + i];
        --at;
      }
      dists[(size_t)at * n_in + i] = d2;
      ids[(size_t)at * n_in + i] = j;
    }
    for (; k < knn; ++k) ids[(size_t)k * n_in + i] = -1, dists[(size_t)k * n_in + i] = INFINITY;
  }
}
