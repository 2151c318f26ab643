// KIE entities that cross tile seams, recovered from a whole-page KIE reading (DESIGN 4.22; include/alm_ocr.h
// alm_omni_merge_kie_whole_page; tile_merge.cu: kie_whole_map_kernel, kie_whole_pair_kernel, kie_whole_compact_kernel).
// whole_core.h's rule (DESIGN 4.17) at entity granularity, on kie_tile_core.h's geometry (DESIGN 4.18).  Like
// tile_core.h the functions compile as host code as well: tests/emu/kie_whole_page_emu.cpp runs them over the whole
// grid without a GPU (test infrastructure only).
//
// The rule, per page p of upright size H x W, read at turn k (0 for upright), tiled with (T, ov) and merged by
// alm_omni_merge_kie_tiles.  Two kinds of entity:
//   tile entities   the merge's output entities of the page, with their words, in page pixels.
//   whole entities  kie_tile_core::walk over the page's whole-page KIE reading: np.rot90(page, k) decoded as one image
//                   through the validation transform.  Word rects kie_tile_core::word_rect with the turned size (tw x
//                   th) and origin 0, i.e. bin_to_coord's image_w * min / num_bins; the entity box is the union of its
//                   words' rects, in the turned frame.
// Each whole entity is decided on its own, by geometry only:
//   keep    iff it has words and every tile of the page's plan cuts its box: tile_core::cut_axis on the box's edges in
//           that tile's frame (edge - origin, exact in double), edges outside the tile included.  A tile cuts the box
//           iff its column cuts it in x or its row cuts it in y, so "some tile does not cut it" holds iff some column
//           passes the x test and some row passes the y test: O(nx + ny) per entity (axis_passes).  A wordless whole
//           entity has no box and is never kept.
//   map     a kept entity's word rects map back to the page corner by corner with tile_core::map_back, min / max
//           re-ordered, its polygons vertex by vertex (kie_tile_core::put_entity on a tile that is the whole turned
//           page); its box maps back the same way, for the test below.
// Each tile entity is decided against the page's kept whole entities:
//   drop    iff its anchor, the centre of its box (the union of its word rects, as DESIGN 4.18's anchor), lies inside the
//           box of a kept whole entity: x0 <= x <= x1 and y0 <= y <= y1, in double, in page pixels (a quarter-turn keeps
//           boxes axis-aligned).  A NaN coordinate is never inside: every comparison with it is false; a non-finite
//           rect coordinate makes the anchor NaN.  A wordless tile entity has no anchor and is never dropped.
//   Trade-off: the test uses the whole entity's box, not its word polygons.  The anchor of a fragment that a tile read
//   of a multi-word entity can fall in a gap between the whole entity's words (two lines of an address, the columns of
//   an invoice line); against the word polygons the fragment would stay beside the whole reading and be read twice.
//   The price: a tile entity whose anchor lies inside a whole entity's box without belonging to it (an entity nested in
//   the gap of a larger one) is dropped.
// Whole entities never drop each other: they are the model's own output.
// Output per page: its kept tile entities in input order, then its kept whole entities in entity order, each with its
// words in decode order (alm_omni_merge_kie_tiles' layout); ent_source = (tile, entity) as the tile merge wrote it for
// tile entities and (-1, entity) for whole ones; word_source = (tile, instance) and (-1, instance).
// Properties (tests/test_kie_whole_page_cpu.py checks each):
//   (a) a whole entity whose box is narrower than ov - 2m in x and shorter than ov - 2m in y is never kept: whole_core.h's
//       argument (a) holds for the box's two edges per axis as it does for a word's vertices.
//   (b) on a page that fits in one tile no whole entity is kept: there is no interior edge, so nothing is cut.
//   (c) the result does not depend on the order of the rows: every decision reads one entity and a set.
#pragma once
#include <math.h>
#include <stdint.h>

#include "kie_tile_core.h"
#include "tile_core.h"

namespace alm {
namespace kie_whole_core {

// the tile a whole-page reading is: page p of upright size H x W read whole at turn k (origin 0, the turned size)
ALM_HD tile_core::Tile whole_tile(int p, int H, int W, int turn) {
  const int T = H > W ? H : W;
  return tile_core::make_turned_tile(p, p, H, W, turn, T, 0, 0, 0.0);
}

// does some tile of the axis (length L of the turned page, tiles (T, ov)) not cut the span [lo, hi] in this axis
ALM_HD bool axis_passes(double lo, double hi, int L, int T, int ov, double m) {
  const int n = tile_core::axis_count(L, T, ov), f = L < T ? L : T;
  for (int i = 0; i < n; ++i) {
    const double o = tile_core::axis_origin(L, T, ov, i);
    const bool a = i > 0, b = i < n - 1;
    if (!(tile_core::cut_axis(quad_core::dadd(lo, -o), a, b, f, m) ||
          tile_core::cut_axis(quad_core::dadd(hi, -o), a, b, f, m)))
      return true;
  }
  return false;
}

// whole entity slot g = page p, entity e (g = p max_ent + e) of kie_whole_map_kernel: keep (1 = every tile of the plan
// cuts its box; 0 also for a wordless entity or an empty slot) and, for a live slot with words, its box [4] mapped to
// the upright page.  wt: the pages' whole tiles (whole_tile); poly: the whole readings, max_inst slots of [32] bins per
// page.
ALM_HD void map_entity(long g, int max_ent, int max_inst, const tile_core::Tile* wt, const int* n_ent,
                       const kie_tile_core::Entity* ents, const int64_t* poly, int T, int ov, int num_bins,
                       double margin, double* box, uint8_t* keep) {
  using tile_core::dmax;
  using tile_core::dmin;
  const int p = static_cast<int>(g / max_ent), e = static_cast<int>(g - static_cast<long>(p) * max_ent);
  if (e >= n_ent[p] || ents[g].words == 0) {
    keep[g] = 0;
    return;
  }
  const tile_core::Tile& t = wt[p];
  const kie_tile_core::Entity& en = ents[g];
  double b[4] = {HUGE_VAL, HUGE_VAL, -HUGE_VAL, -HUGE_VAL};  // in the turned frame
  for (int k = 0; k < en.words; ++k) {
    double r[4];
    kie_tile_core::word_rect(poly + (static_cast<long>(p) * max_inst + en.first + k) * 32, t.w, t.h, num_bins, r);
    b[0] = dmin(b[0], r[0]); b[1] = dmin(b[1], r[1]);
    b[2] = dmax(b[2], r[2]); b[3] = dmax(b[3], r[3]);
  }
  keep[g] = !(axis_passes(b[0], b[2], t.w, T, ov, margin) && axis_passes(b[1], b[3], t.h, T, ov, margin));
  double x0, y0, x1, y1;
  const double H = t.ph, W = t.pw;
  tile_core::map_back(t.turn, b[0], b[1], H, W, &x0, &y0);
  tile_core::map_back(t.turn, b[2], b[3], H, W, &x1, &y1);
  box[4 * g] = dmin(x0, x1);
  box[4 * g + 1] = dmin(y0, y1);
  box[4 * g + 2] = dmax(x0, x1);
  box[4 * g + 3] = dmax(y0, y1);
}

// the anchor (x, y) of a tile entity whose n >= 1 word rects [4] start at rects: the centre of their union, NaN when a
// coordinate is not finite
ALM_HD void anchor(const double* rects, int n, double* x, double* y) {
  using quad_core::dadd;
  using tile_core::dmax;
  using tile_core::dmin;
  double b[4] = {HUGE_VAL, HUGE_VAL, -HUGE_VAL, -HUGE_VAL}, nf = 0.0;
  for (int k = 0; k < n; ++k) {
    const double* r = rects + 4 * k;
    b[0] = dmin(b[0], r[0]); b[1] = dmin(b[1], r[1]);
    b[2] = dmax(b[2], r[2]); b[3] = dmax(b[3], r[3]);
    nf = dadd(nf, dadd(dadd(dadd(r[0], -r[0]), dadd(r[1], -r[1])), dadd(dadd(r[2], -r[2]), dadd(r[3], -r[3]))));
  }
  *x = dadd(quad_core::dmul(dadd(b[0], b[2]), 0.5), nf);
  *y = dadd(quad_core::dmul(dadd(b[1], b[3]), 0.5), nf);
}

// is (x, y) inside the box b (x0, y0, x1, y1), edges included
ALM_HD bool inside(double x, double y, const double* b) { return b[0] <= x && x <= b[2] && b[1] <= y && y <= b[3]; }

// kept tile entity n goes to entity row o, its words to word rows wo ..: every field copied, the word rows moved
ALM_HD void put_tile(long n, long o, long wo, const int* cls, const float* prob, const int* word_offset,
                     const int* word_count, const int* ent_src, const double* rects, const double* polys,
                     const int* word_src, int* cls_out, float* prob_out, int* word_offset_out, int* word_count_out,
                     int* ent_src_out, double* rects_out, double* polys_out, int* word_src_out) {
  const int nw = word_count[n];
  cls_out[o] = cls[n];
  prob_out[o] = prob[n];
  word_offset_out[o] = static_cast<int>(wo);
  word_count_out[o] = nw;
  ent_src_out[2 * o] = ent_src[2 * n];
  ent_src_out[2 * o + 1] = ent_src[2 * n + 1];
  for (int k = 0; k < nw; ++k) {
    const long w = static_cast<long>(word_offset[n]) + k, v = wo + k;
    for (int j = 0; j < 4; ++j) rects_out[4 * v + j] = rects[4 * w + j];
    for (int j = 0; j < 32; ++j) polys_out[32 * v + j] = polys[32 * w + j];
    word_src_out[2 * v] = word_src[2 * w];
    word_src_out[2 * v + 1] = word_src[2 * w + 1];
  }
}

// kept whole entity slot g goes to entity row o, its words to word rows wo ..: kie_tile_core::put_entity on the page's
// whole tile, sources (-1, entity) and (-1, instance)
ALM_HD void put_whole(long g, long o, long wo, int max_ent, int max_inst, const tile_core::Tile* wt,
                      const kie_tile_core::Entity* ents, const int64_t* poly, int num_bins, int* cls_out,
                      float* prob_out, int* word_offset, int* word_count, int* ent_src, double* rects, double* polys,
                      int* word_src) {
  kie_tile_core::put_entity(g, o, wo, max_ent, max_inst, wt, ents, poly, num_bins, cls_out, prob_out, word_offset,
                            word_count, ent_src, rects, polys, word_src);
  ent_src[2 * o] = -1;
  for (int k = 0; k < ents[g].words; ++k) word_src[2 * (wo + k)] = -1;
}

}  // namespace kie_whole_core
}  // namespace alm
