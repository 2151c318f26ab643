// TEST INFRASTRUCTURE: host emulation of the recovery of KIE entities that cross tile seams (DESIGN 4.22).  Compiles the
// bodies shared with the CUDA kernels (advancedliteratemachinery_b200/csrc/kie_whole_core.h, kie_tile_core.h,
// tile_core.h) as plain C++ and runs them over the whole grid of each launch: the host walk that builds the whole entity
// table, kie_whole_map_kernel, kie_whole_pair_kernel and kie_whole_compact_kernel in (page, tile entities, whole slots)
// order.  Built on the fly by tests/test_kie_whole_page_cpu.py (g++ -O1 -ffp-contract=off); never part of
// libalm_ocr.so.
#include <stdint.h>

#include <vector>

#include "../../advancedliteratemachinery_b200/csrc/kie_tile_core.h"
#include "../../advancedliteratemachinery_b200/csrc/kie_whole_core.h"
#include "../../advancedliteratemachinery_b200/csrc/tile_core.h"

using namespace alm;

extern "C" {

// alm_omni_merge_kie_whole_page on the host (turns null = upright; layout and counts validated by the caller): returns
// the number of kept entities and writes the kept word count to *n_words, or -1 when a whole reading fails the walk
long emu_merge_kie_whole_page(const int* heights, const int* widths, const int* turns, int n_pages, int T, int ov,
                              double margin, int num_bins, int class_base, int n_classes, const int* count,
                              const int* offset, const int* cls, const float* prob, const int* word_offset,
                              const int* word_count, const int* ent_src, const double* rects, const double* polys,
                              const int* word_src, const int* n_tok, const int64_t* tokens, const float* tok_prob,
                              int max_tok, const int* n_inst, const int32_t* inst_pos, const int64_t* poly,
                              int max_inst, int* page_count, int* page_offset, int* cls_out, float* prob_out,
                              int* woff_out, int* wcnt_out, int* src_out, double* rects_out, double* polys_out,
                              int* wsrc_out, long* n_words) {
  std::vector<tile_core::Tile> wt;
  for (int p = 0; p < n_pages; ++p) wt.push_back(kie_whole_core::whole_tile(p, heights[p], widths[p], turns ? turns[p] : 0));
  std::vector<std::vector<kie_tile_core::Entity>> per(n_pages);
  std::vector<int> n_ent(n_pages);
  int max_ent = 1;
  for (int p = 0; p < n_pages; ++p) {  // the host walk
    int pairs = 0;
    const long o = static_cast<long>(p) * max_tok;
    if (kie_tile_core::walk(tokens + o, tok_prob + o, n_tok[p], inst_pos + static_cast<long>(p) * max_inst, n_inst[p],
                            num_bins, class_base, n_classes, &per[p], &pairs) != kie_tile_core::kWalkOk ||
        pairs != n_inst[p])
      return -1;
    n_ent[p] = static_cast<int>(per[p].size());
    max_ent = n_ent[p] > max_ent ? n_ent[p] : max_ent;
  }
  const long S = static_cast<long>(n_pages) * max_ent;
  std::vector<kie_tile_core::Entity> ents(S, kie_tile_core::Entity{0, 0.f, 0, 0});
  for (int p = 0; p < n_pages; ++p)
    for (int e = 0; e < n_ent[p]; ++e) ents[static_cast<long>(p) * max_ent + e] = per[p][e];
  std::vector<double> box(S * 4);
  std::vector<uint8_t> keep(S);
  for (long g = 0; g < S; ++g)  // kie_whole_map_kernel
    kie_whole_core::map_entity(g, max_ent, max_inst, wt.data(), n_ent.data(), ents.data(), poly, T, ov, num_bins,
                               margin, box.data(), keep.data());
  long o = 0, w = 0;  // kie_whole_pair_kernel + kie_whole_compact_kernel
  for (int p = 0; p < n_pages; ++p) {
    page_offset[p] = static_cast<int>(o);
    for (long n = offset[p]; n < static_cast<long>(offset[p]) + count[p]; ++n) {
      bool dropped = false;
      if (word_count[n] > 0) {
        double ax, ay;
        kie_whole_core::anchor(rects + 4L * word_offset[n], word_count[n], &ax, &ay);
        for (int e = 0; e < n_ent[p] && !dropped; ++e) {
          const long g = static_cast<long>(p) * max_ent + e;
          dropped = keep[g] && kie_whole_core::inside(ax, ay, &box[4 * g]);
        }
      }
      if (dropped) continue;
      kie_whole_core::put_tile(n, o++, w, cls, prob, word_offset, word_count, ent_src, rects, polys, word_src, cls_out,
                               prob_out, woff_out, wcnt_out, src_out, rects_out, polys_out, wsrc_out);
      w += word_count[n];
    }
    for (int e = 0; e < n_ent[p]; ++e) {
      const long g = static_cast<long>(p) * max_ent + e;
      if (!keep[g]) continue;
      kie_whole_core::put_whole(g, o++, w, max_ent, max_inst, wt.data(), ents.data(), poly, num_bins, cls_out,
                                prob_out, woff_out, wcnt_out, src_out, rects_out, polys_out, wsrc_out);
      w += ents[g].words;
    }
    page_count[p] = static_cast<int>(o - page_offset[p]);
  }
  *n_words = w;
  return o;
}

}  // extern "C"
