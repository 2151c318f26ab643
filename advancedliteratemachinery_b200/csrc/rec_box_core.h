// Character boxes in page pixels from the recognition loop's character locations of words read in tiles, turned or
// not (DESIGN 4.20; include/alm_ocr.h alm_omni_char_boxes; tile_merge.cu: rec_box_kernel).  Like tile_core.h the
// functions compile as host code as well: tests/emu/rec_box_emu.cpp runs them without a GPU (test infrastructure only).
//
// The rule.  A word: its 16-vertex polygon P in page pixels (what the merges and read_regions return, vertex order kept:
// P_0..P_7 the top boundary in the reading direction, P_8..P_15 the bottom one back), its rec ids [L] and the locations
// [L][5] = (cx, cy, sxx, sxy, syy) of the tile instance it came from, normalised by that image's encoded size.  Its
// frame: the upright page size H x W, the turn k and the tile's origin (y0, x0) and size h x w in the turned page (a
// page read whole: origin 0, the page's size, turn 0).  Every operation in double, rounded on its own.
//   centre  (u, v) = (x0 + cx w, y0 + cy h), then tile_core::map_back(k, u, v, H, W): the map the merges apply to
//           points and vertices, so centres and polygons cannot disagree.
//   cov     Sigma_t = (sxx w w, sxy w h, syy h h), then R Sigma_t R^T with R the linear part of map_back: an odd k swaps
//           sxx and syy and negates sxy, k = 2 leaves Sigma unchanged.
//   chars   decode_seq's walk over the steps in order (utils/misc.py:162-184): stop at recog_pad or rec_eos, skip
//           recog_pad - 1.  Character i is the i-th kept step.
//   box     postprocess.rec_char_boxes' rule on P: centre line c_i = (P_i + P_{15-i}) / 2 and local height h_i =
//           |P_i - P_{15-i}|, i = 0..7; q = the point of the polyline c_0..c_7 nearest the centre mu (parameter s on
//           segment i clipped to [0, 1], s = 0 on a zero-length segment; the first minimum, or the first NaN distance,
//           as np.argmin picks); u = the unit direction of segment i (zero length: c_7 - c_0; also zero: (1, 0)), v =
//           (-u_y, u_x); height H_q = h_i + s (h_{i+1} - h_i); half-width a = sqrt(3) sqrt(max(u^T Sigma u, 0));
//           corners q - a u - (H_q / 2) v, q + a u - (H_q / 2) v, q + a u + (H_q / 2) v, q - a u + (H_q / 2) v.
//           Lengths are sqrt(x x + y y), not hypot, so the device and a host build agree bit for bit.
// Non-finite inputs propagate as NaN through the same arithmetic; they are never an error.
#pragma once
#include <math.h>
#include <stdint.h>

#include "tile_core.h"

namespace alm {
namespace rec_box_core {

constexpr int kMaxSteps = 1021;  // rec_length's upper bound (alm_omni_decode)

// one tile or whole page a word was read in
struct Frame {
  int H, W, turn;    // the upright page and the turn it was read at
  int y0, x0, h, w;  // the tile in the turned page
};

// positive sizes, a turn in 0..3 and the tile inside the turned page
ALM_HD bool valid_frame(const Frame& f) {
  if (f.H < 1 || f.W < 1 || f.h < 1 || f.w < 1 || f.turn < 0 || f.turn > 3 || f.y0 < 0 || f.x0 < 0) return false;
  const long th = f.turn & 1 ? f.W : f.H, tw = f.turn & 1 ? f.H : f.W;
  return static_cast<long>(f.y0) + f.h <= th && static_cast<long>(f.x0) + f.w <= tw;
}

enum { kKeep = 0, kSkip = 1, kStop = 2 };

// decode_seq's walk: what step id tok does to the character string
ALM_HD int step_kind(int64_t tok, int64_t pad, int64_t eos) {
  if (tok == pad || tok == eos) return kStop;
  return tok == pad - 1 ? kSkip : kKeep;
}

ALM_HD double length(double x, double y) {
  using quad_core::dadd;
  using quad_core::dmul;
  return sqrt(dadd(dmul(x, x), dmul(y, y)));
}

// centre-line point i (0..7) of polygon P [32]
ALM_HD void centre_point(const double* P, int i, double* x, double* y) {
  using quad_core::dadd;
  using quad_core::ddiv;
  *x = ddiv(dadd(P[2 * i], P[2 * (15 - i)]), 2.0);
  *y = ddiv(dadd(P[2 * i + 1], P[2 * (15 - i) + 1]), 2.0);
}

// local height i (0..7) of polygon P
ALM_HD double height(const double* P, int i) {
  using quad_core::dadd;
  return length(dadd(P[2 * i], -P[2 * (15 - i)]), dadd(P[2 * i + 1], -P[2 * (15 - i) + 1]));
}

// one character: its location loc [5] in frame f, the word's page polygon P [32] -> centre [2], cov [3] (sxx, sxy,
// syy) and box [8] (four corners (x, y)) in page pixels
ALM_HD void char_box(const double* P, const Frame& f, const float* loc, double* centre, double* cov, double* box) {
  using quad_core::dadd;
  using quad_core::ddiv;
  using quad_core::dmul;
  const double w = f.w, h = f.h;
  double mx, my;
  tile_core::map_back(f.turn, dadd(f.x0, dmul(loc[0], w)), dadd(f.y0, dmul(loc[1], h)), f.H, f.W, &mx, &my);
  double sxx = dmul(dmul(loc[2], w), w), sxy = dmul(dmul(loc[3], w), h), syy = dmul(dmul(loc[4], h), h);
  if (f.turn & 1) {
    const double t = sxx;
    sxx = syy;
    syy = t;
    sxy = -sxy;
  }
  centre[0] = mx;
  centre[1] = my;
  cov[0] = sxx;
  cov[1] = sxy;
  cov[2] = syy;
  // the nearest point of the centre line: segment bi at parameter bs
  int bi = 0;
  double best = 0.0, bs = 0.0;
  double ax, ay;
  centre_point(P, 0, &ax, &ay);
  for (int i = 0; i < 7; ++i) {
    double bx, by;
    centre_point(P, i + 1, &bx, &by);
    const double sx = dadd(bx, -ax), sy = dadd(by, -ay);
    const double seg2 = dadd(dmul(sx, sx), dmul(sy, sy));
    double s = 0.0;
    if (seg2 > 0.0) {
      s = ddiv(dadd(dmul(dadd(mx, -ax), sx), dmul(dadd(my, -ay), sy)), seg2);
      s = s < 0.0 ? 0.0 : s;  // NaN passes, as np.clip lets it
      s = s > 1.0 ? 1.0 : s;
    }
    const double dx = dadd(mx, -dadd(ax, dmul(s, sx))), dy = dadd(my, -dadd(ay, dmul(s, sy)));
    const double d = dadd(dmul(dx, dx), dmul(dy, dy));
    if (i == 0 || (best == best && (d != d || d < best))) {  // np.argmin: the first NaN, else the first minimum
      best = d;
      bi = i;
      bs = s;
    }
    ax = bx;
    ay = by;
  }
  double cx, cy, nx, ny;
  centre_point(P, bi, &cx, &cy);
  centre_point(P, bi + 1, &nx, &ny);
  double dx = dadd(nx, -cx), dy = dadd(ny, -cy);
  const double qx = dadd(cx, dmul(bs, dx)), qy = dadd(cy, dmul(bs, dy));
  if (!(dadd(dmul(dx, dx), dmul(dy, dy)) > 0.0)) {  // a zero-length segment: the chord c_7 - c_0
    double x0, y0, x7, y7;
    centre_point(P, 0, &x0, &y0);
    centre_point(P, 7, &x7, &y7);
    dx = dadd(x7, -x0);
    dy = dadd(y7, -y0);
  }
  const double norm = length(dx, dy);
  const double ux = norm > 0.0 ? ddiv(dx, norm) : 1.0, uy = norm > 0.0 ? ddiv(dy, norm) : 0.0;
  const double vx = -uy, vy = ux;
  const double h0 = height(P, bi);
  const double hq = dadd(h0, dmul(bs, dadd(height(P, bi + 1), -h0)));
  double var = dadd(dadd(dmul(dmul(ux, ux), sxx), dmul(dmul(dmul(2.0, ux), uy), sxy)), dmul(dmul(uy, uy), syy));
  var = 0.0 > var ? 0.0 : var;  // max(var, 0.0): NaN passes
  const double a = dmul(sqrt(3.0), sqrt(var)), half = ddiv(hq, 2.0);
  const double aux = dmul(a, ux), auy = dmul(a, uy), hvx = dmul(half, vx), hvy = dmul(half, vy);
  box[0] = dadd(dadd(qx, -aux), -hvx);
  box[1] = dadd(dadd(qy, -auy), -hvy);
  box[2] = dadd(dadd(qx, aux), -hvx);
  box[3] = dadd(dadd(qy, auy), -hvy);
  box[4] = dadd(dadd(qx, aux), hvx);
  box[5] = dadd(dadd(qy, auy), hvy);
  box[6] = dadd(dadd(qx, -aux), hvx);
  box[7] = dadd(dadd(qy, -auy), hvy);
}

}  // namespace rec_box_core
}  // namespace alm
