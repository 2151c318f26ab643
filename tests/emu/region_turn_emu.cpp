// TEST INFRASTRUCTURE: host emulation of the choice among a region's turned readings (DESIGN 4.21).  Compiles the
// bodies shared with the CUDA kernel (advancedliteratemachinery_b200/csrc/region_turn_core.h) as plain C++ and runs
// region_select_kernel's work region by region: each candidate's fuse_core::spot_score (the kernel adds the same
// probabilities in the same order from shuffles), region_turn_core::pick, and the kept reading's 17 points mapped to
// the page.  Built on the fly by tests/test_region_turns_cpu.py (g++ -O1 -ffp-contract=off); never part of
// libalm_ocr.so.
#include <stdint.h>

#include <vector>

#include "../../advancedliteratemachinery_b200/csrc/region_turn_core.h"

using namespace alm;

extern "C" {

// alm_omni_select_regions on the host (arguments validated by the caller)
void emu_select_regions(long R, int C, const int* frame_index, int F, const int* frames, const int64_t* pt,
                        const int64_t* poly, const int64_t* rec, const float* prob, int L, int num_bins, int64_t pad,
                        int64_t eos, int* kept, double* scores, double* pts, double* polys) {
  std::vector<region_turn_core::Frame> fr(F);
  for (int k = 0; k < F; ++k) {
    const int* v = frames + 7L * k;
    fr[k] = region_turn_core::Frame{v[0], v[1], v[2], v[3], v[4], v[5], v[6]};
  }
  for (long r = 0; r < R; ++r) {
    double s[region_turn_core::kMaxCandidates];
    int k[region_turn_core::kMaxCandidates];
    for (int c = 0; c < C; ++c) {
      const long g = r * C + c;
      s[c] = fuse_core::spot_score(rec + g * L, prob + g * L, L, pad, eos);
      k[c] = fr[frame_index[g]].turn;
      scores[g] = s[c];
    }
    const int best = region_turn_core::pick(s, k, C);
    kept[r] = best;
    const long g = r * C + best;
    for (int i = 0; i < 17; ++i)
      region_turn_core::map_row_point(fr[frame_index[g]], pt + 2 * g, poly + 32 * g, i, num_bins,
                                      i == 0 ? pts + 2 * r : polys + 32 * r + 2 * (i - 1));
  }
}

}  // extern "C"
