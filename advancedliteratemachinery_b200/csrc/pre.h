// Test-time image pipeline (preproc.cu): shared declarations.
#pragma once
#include <algorithm>
#include <vector>

#include "alm_internal.h"
#include "group_core.h"
#include "kie_tile_core.h"
#include "kie_whole_core.h"
#include "rec_box_core.h"
#include "tile_core.h"
#include "whole_core.h"

namespace alm {

// Host <-> device staging of one call on the context's stream, in workspace buffers released when the call ends.
// Every buffer gets at least one element, so an empty one is still a valid pointer, and empty copies are skipped.
class Staging {
 public:
  explicit Staging(Ctx* c) : c_(c), scope_(ready(c)) {}
  // a device buffer of n elements
  template <class T>
  T* out(size_t n) {
    return c_->ws.get<T>(std::max<size_t>(n, 1));
  }
  // a device copy of host src [n]; src must stay valid until the next sync()
  template <class T>
  const T* up(const T* src, size_t n) {
    T* d = out<T>(n);
    if (n) ALM_CHECK_CUDA(cudaMemcpyAsync(d, src, n * sizeof(T), cudaMemcpyHostToDevice, c_->stream));
    return d;
  }
  // host dst [n] from device src, complete after the next sync()
  template <class T>
  void down(T* dst, const T* src, size_t n) {
    if (n) ALM_CHECK_CUDA(cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyDeviceToHost, c_->stream));
  }
  void sync() { ALM_CHECK_CUDA(cudaStreamSynchronize(c_->stream)); }

 private:
  static Arena& ready(Ctx* c) {
    c->ensure_ws();
    return c->ws;
  }
  Ctx* c_;
  ArenaScope scope_;
};

// Host outputs of the row merges (tile_merge, reading_merge, whole_merge): per page its kept row count and its first
// kept row [n_pages], then the kept rows in page order, each pts [2], polys [32], rec [L], prob [L] and source [2].
// The row buffers hold at least the merge's input rows.
struct MergeRows {
  int* page_count;
  int* page_offset;
  double* pts;
  double* polys;
  int64_t* rec;
  float* prob;
  int* source;
};

enum { PRE_BILINEAR = 0, PRE_BICUBIC = 1 };

struct PreImage {
  const uint8_t* dev_rgb;  // device, [h][w][3] uint8
  int h, w;                // source size
  int oh, ow;              // resized size
};

// RandomResize.get_size_with_aspect_ratio for one (h, w) (host only)
void pre_omni_size(int h, int w, int min_size, int max_size, int* oh, int* ow);
// fixed-point weights of one pass: bounds [out][2], coefs [out][*ksize] (call with coefs == nullptr to size the buffers)
int pre_coeffs(int in_size, int out_size, int filter, int* ksize, int* bounds, int* coefs, size_t cap_ints);
// the same weights appended to `host` as bounds [out][2] then coefs [out][ksize]; returns ksize
int pre_append_coeffs(int in_size, int out_size, int filter, std::vector<int>* host);
// Resize every image with Pillow's 8-bit resampling, ToTensor (+ Normalize), write it into the top-left corner of its
// [3, Hc, Wc] slot of `out` (zero elsewhere) and, optionally, the pad mask [n, Hc, Wc] (1 = padding).
void pre_resize_batch(Ctx* c, const std::vector<PreImage>& imgs, int filter, bool normalize, float* out, int Hc, int Wc,
                      uint8_t* mask);

// Perspective crops of detected text regions (quadcrop.cu): DocXChain's TextRecognition.order_point + crop_image
// (Applications/DocXChain/modules/text_recognition.py:84-145) per region, host part.
struct QuadPlan {
  float ordered[8];  // order_point's result
  float corners[8];  // crop_image's source corners (the getPerspectiveTransform input)
  int cw, ch;        // crop width / height (the page's size when either truncated distance is 0)
  double mi[9];      // inverse of the perspective transform: crop pixel -> page coordinates
  int page;
};
// plans of R regions, quads f32 [R][4][2] on pages heights / widths; throws AlmError(ALM_ERR_INVALID) naming the region
std::vector<QuadPlan> pre_quad_plan(const int* heights, const int* widths, int n_pages, const float* quads,
                                    const int* page_index, int R);
// warp every planned region out of its page, Pillow-bicubic resize it to imgW x imgH and ToTensor it into
// out [R][3][imgH][imgW] (device): three launches whatever R is.  turns: host [R] (0..3, quad_core::unturn), or null
// for upright crops
void pre_quad_crops(Ctx* c, const std::vector<PreImage>& pages, const std::vector<QuadPlan>& plans, int imgH, int imgW,
                    float* out, const int* turns = nullptr);

// Curved text (quadcrop.cu): OmniParser's 16-point polygon (8 points of the top boundary left -> right, then 8 of the
// bottom one right -> left) rectified along the cubic Beziers fitted to both boundaries, host part.
struct CurvePlan {
  double ctrl[2][4][2];  // top, bottom: control points (x, y)
  int cw, ch;            // crop width / height, at least 1 x 1
  int page;
};
// plans of R regions, polys f32 [R][16][2]; throws AlmError(ALM_ERR_INVALID) naming the region
std::vector<CurvePlan> pre_curve_plan(const int* heights, const int* widths, int n_pages, const float* polys,
                                      const int* page_index, int R);
// rectify every planned region, Pillow-bicubic resize it to imgW x imgH and ToTensor it into out [R][3][imgH][imgW]
// (device): three launches whatever R is; turns as pre_quad_crops
void pre_curve_crops(Ctx* c, const std::vector<PreImage>& pages, const std::vector<CurvePlan>& plans, int imgH, int imgW,
                     float* out, const int* turns = nullptr);

// Long text lines (line_core.h): every window of every planned region, in region order, cut from the region's full
// crop, Pillow-bicubic resized to 128 x 32 and ToTensor'ed into out [sum of windows][3][32][128] (device): three
// launches whatever the number of regions.  turns as pre_quad_crops: the windows are laid out on the turned crop.
void pre_line_crops(Ctx* c, const std::vector<PreImage>& pages, const std::vector<QuadPlan>& plans, float* out,
                    const int* turns = nullptr);
void pre_line_crops(Ctx* c, const std::vector<PreImage>& pages, const std::vector<CurvePlan>& plans, float* out,
                    const int* turns = nullptr);

// Pages spotted in tiles (tile_core.h, tile_merge.cu): merge the decoded instances of `tiles` (the plan's tiles of every
// page in plan order; max_inst slots each, the layout of alm_omni_decode, host buffers) into page coordinates.  Writes
// the page counts and offsets and the kept rows (page then tile then instance order) to out, whose rows hold at least
// sum(n_inst).  Three launches whatever the page and tile counts.
void tile_merge(Ctx* c, const std::vector<tile_core::Tile>& tiles, int n_pages, int max_inst, int L, int num_bins,
                double margin, double iou, const int* n_inst, const int64_t* pt, const int64_t* poly, const int64_t* rec,
                const float* prob, const MergeRows& out);

// Turned pages (page_turn.cu, DESIGN 4.14).  tile_gather: tiles idx[0], idx[1], ... of `tiles` (make_tile /
// make_turned_tile of the staged `pages`) cut into one workspace buffer, [h][w][3] each, in one launch; imgs gets one
// PreImage per tile (oh / ow unset).  orient_select: per page the scores f64 [n_pages][4] of its four readings (host
// decode outputs of 4 n_pages readings in the layout of alm_omni_decode, reading 4 p + k = page p at turn k) and the
// chosen turn [n_pages], both written to the host; one launch.
void tile_gather(Ctx* c, const std::vector<PreImage>& pages, const std::vector<tile_core::Tile>& tiles,
                 const std::vector<int>& idx, std::vector<PreImage>* imgs);
void orient_select(Ctx* c, int n_pages, int max_inst, int L, int64_t pad, int64_t eos, const int* n_inst,
                   const int64_t* rec, const float* prob, int* turns_out, double* scores);
// Caller-given regions read at quarter-turns (page_turn.cu; rule: region_turn_core.h, DESIGN 4.21).  Host inputs: R
// regions of C candidate readings, frame_index [R][C] into frames [F] (checked by the caller), read_at's pt [R][C][2],
// poly [R][C][32], rec / prob [R][C][L].  Host outputs: kept [R], scores [R][C], the kept reading's pts [R][2] and polys
// [R][32] in upright page pixels.  One launch; none when R = 0.
void region_select(Ctx* c, long R, int C, int L, int F, const rec_box_core::Frame* frames, const int* frame_index,
                   const int64_t* pt, const int64_t* poly, const int64_t* rec, const float* prob, int num_bins,
                   int64_t pad, int64_t eos, int* kept, double* scores, double* pts, double* polys);

// A page's nr readings merged into one set of words (tile_merge.cu; rule: turn_core.h): its four turned readings
// (nr = 4, DESIGN 4.15) or a dense page's window readings (DESIGN 4.16).  Host inputs in the layout
// alm_omni_merge_tiles_turned writes for nr n_pages readings (reading nr p + k = page p's reading k; count / offset
// [nr n_pages], offsets the exclusive prefix of the counts, checked by the caller); out as tile_merge's, source = (k,
// index within the reading).  Three launches.
void reading_merge(Ctx* c, int n_pages, int nr, const int* count, const int* offset, int L, int64_t pad, int64_t eos,
                   double iou, const double* pts, const double* polys, const int64_t* rec, const float* prob,
                   const MergeRows& out);

// Words that cross tile seams, recovered from a whole-page reading of each page (tile_merge.cu; rule: whole_core.h,
// DESIGN 4.17).  Host inputs: the tile merge's rows of the pages (count / offset [n_pages], offsets the exclusive
// prefix of the counts, checked by the caller; pts, polys, rec, prob, src in the layout alm_omni_merge_tiles writes) and
// the whole-page readings in the layout of alm_omni_decode with cap slots per page (n_inst [n_pages] in [0, cap]).
// The rows of out hold at least sum(count) + sum(n_inst).  Three launches.
void whole_merge(Ctx* c, const std::vector<whole_core::Page>& pages, int T, int ov, int num_bins, double margin,
                 int L, const int* count, const int* offset, const double* pts, const double* polys,
                 const int64_t* rec, const float* prob, const int* src, int cap, const int* n_inst, const int64_t* pt,
                 const int64_t* poly, const int64_t* wrec, const float* wprob, const MergeRows& out);

// KIE entities of pages read in tiles, turned or not (tile_merge.cu; rule: kie_tile_core.h, DESIGN 4.18).  Host
// inputs: the entity table of every tile (max_ent slots per tile, n_ent [tiles] used; kie_tile_core::walk's rows, checked
// by the caller) and the tiles' polygons in the layout of alm_omni_decode_kie (max_inst slots of [32] bins per tile).
// Writes page_count / page_offset [n_pages], the kept entities (page, tile, entity order) and their words to the host
// outputs, which hold every entity and every entity's words.  Four launches whatever the counts.
void kie_merge(Ctx* c, const std::vector<tile_core::Tile>& tiles, int n_pages, int max_ent, const int* n_ent,
               const kie_tile_core::Entity* ents, int max_inst, const int64_t* poly, int num_bins, double margin,
               double iou, int* page_count, int* page_offset, int* cls_out, float* prob_out, int* word_offset,
               int* word_count, int* ent_src, double* rects, double* polys, int* word_src);

// KIE entities that cross tile seams, recovered from a whole-page KIE reading of each page (tile_merge.cu; rule:
// kie_whole_core.h, DESIGN 4.22).  Host inputs: wt, each page's whole tile (kie_whole_core::whole_tile); the KIE tile
// merge's output of the pages (count / offset [n_pages] and word_offset / word_count [E] exclusive prefixes, checked by
// the caller; cls, prob, ent_src, rects, polys, word_src in the layout alm_omni_merge_kie_tiles writes); the whole
// readings' entity table (max_ent slots per page, n_ent [n_pages] used; kie_tile_core::walk's rows) and polygons
// (max_inst slots of [32] bins per page).  Writes page_count / page_offset [n_pages], the kept entities (page order;
// tile entities, then whole ones) and their words to the host outputs, which hold every input entity and every word.
// Three launches whatever the counts.
void kie_whole_merge(Ctx* c, const std::vector<tile_core::Tile>& wt, int T, int ov, int num_bins, double margin,
                     const int* count, const int* offset, const int* cls, const float* prob, const int* word_offset,
                     const int* word_count, const int* ent_src, const double* rects, const double* polys,
                     const int* word_src, int max_ent, const int* n_ent, const kie_tile_core::Entity* ents,
                     int max_inst, const int64_t* poly, int* page_count, int* page_offset, int* cls_out,
                     float* prob_out, int* woff_out, int* wcnt_out, int* src_out, double* rects_out, double* polys_out,
                     int* wsrc_out);

// Character boxes in page pixels (tile_merge.cu; rule: rec_box_core.h, DESIGN 4.20).  Host inputs: N words' page
// polygons [N][32], rec ids [N][L], locations [N][L][5] and frame index [N] (into frames [F], checked by the caller).
// Host outputs: n_chars [N] and per slot [N][L] the step, centre [2], cov [3] and box [8]; slots past n_chars are 0.
// One launch; none when N = 0.
void char_boxes(Ctx* c, long N, int L, int F, const rec_box_core::Frame* frames, const int* frame_index,
                const double* polys, const int64_t* rec, const float* loc, int64_t pad, int64_t eos, int* n_chars,
                int* step, double* centre, double* cov, double* box);

// Words -> text lines (group_core.h, line_group.cu): the N word polygons f64 [N][32] of n_pages pages (page p = rows
// page_offset[p] .. + page_count[p] - 1, the rows of all pages partition [0, N); host buffers) grouped into lines.
// Writes n_lines / line_offset [n_pages], line_first / line_words / line_polys [lines], order / line_of / rank_of [N]
// to the host outputs.  Five launches whatever the counts; none when N = 0.
void group_lines(Ctx* c, int n_pages, const int* page_count, const int* page_offset, long N, const double* polys,
                 const group_core::Params& prm, int* n_lines, int* line_offset, int* line_first, int* line_words,
                 int* order, int* line_of, int* rank_of, double* line_polys);

}  // namespace alm
