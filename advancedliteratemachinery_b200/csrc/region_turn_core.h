// Caller-given regions read at quarter-turns: of each region's candidate readings, the one kept and its point and
// polygon in upright page pixels (DESIGN 4.21; include/alm_ocr.h alm_omni_select_regions; page_turn.cu:
// region_select_kernel).  Like tile_core.h the functions compile as host code as well: tests/emu/region_turn_emu.cpp
// runs them without a GPU (test infrastructure only).
//
// The rule.  Region r has C (1..4) candidate readings, c = 0 .. C - 1, each read_at's point bins [2], polygon bins [32]
// and rec ids / probabilities [L] of the region read in one frame (rec_box_core::Frame: the upright page H x W, the
// turn k the page was read at, the tile's origin (y0, x0) and size h x w in the turned page; a page read whole has
// origin 0 and the turned page's size).
//   score   s_c = fuse_core::spot_score of the candidate's rec / prob: decode_pred_seq's 'score', in double.
//   keep    the candidate of the largest score; on equal scores the lower turn, then the lower index.  A NaN score
//           never ranks above another reading and every other reading ranks above it (turn_core.h's order), so a NaN
//           is kept only when every candidate's score is NaN, and then candidate 0.
//   map     each of the kept candidate's 17 points (the point, then the 16 vertices in order): the tile merge's
//           mapping, x0 + f32(f32(id / num_bins) * w) with the sum in double (y: y0 and h), then
//           tile_core::map_back(k, ., H, W), one double operation per coordinate.  Turn 0 with one candidate gives
//           omniparser.tile_to_page's values bit for bit; vertex order is kept.
#pragma once
#include <stdint.h>

#include "fuse_core.h"
#include "rec_box_core.h"
#include "tile_core.h"

namespace alm {
namespace region_turn_core {

constexpr int kMaxCandidates = 4;

using rec_box_core::Frame;

// does a reading of score sb at turn kb rank above one of score sa at turn ka (equal turns: neither does)
ALM_HD bool ranks_above(double sb, int kb, double sa, int ka) {
  if (sb != sb) return false;  // NaN never ranks above
  if (sa != sa) return true;   // and every number ranks above NaN
  if (sb != sa) return sb > sa;
  return kb < ka;
}

// which of C candidates (scores s, turns k) is kept: the first that no other ranks above
ALM_HD int pick(const double* s, const int* k, int C) {
  int best = 0;
  for (int c = 1; c < C; ++c)
    if (ranks_above(s[c], k[c], s[best], k[best])) best = c;
  return best;
}

// bins (ix, iy) of a reading in frame f -> upright page pixels
ALM_HD void map_point(const Frame& f, int64_t ix, int64_t iy, int num_bins, double* x, double* y) {
  using quad_core::dadd;
  const double u = dadd(f.x0, static_cast<double>(tile_core::bin_to_coord(ix, num_bins, f.w)));
  const double v = dadd(f.y0, static_cast<double>(tile_core::bin_to_coord(iy, num_bins, f.h)));
  tile_core::map_back(f.turn, u, v, f.H, f.W, x, y);
}

// point i (0: the prompt point pt [2]; 1..16: vertex i - 1 of poly [32]) of a reading in frame f -> out [2]
ALM_HD void map_row_point(const Frame& f, const int64_t* pt, const int64_t* poly, int i, int num_bins, double* out) {
  const int64_t* b = i == 0 ? pt : poly + 2 * (i - 1);
  map_point(f, b[0], b[1], num_bins, &out[0], &out[1]);
}

}  // namespace region_turn_core
}  // namespace alm
